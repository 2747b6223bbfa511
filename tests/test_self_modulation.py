"""Self-modulated batch norm (reference arch_ops.py:370-420): `G.batch_norm_fn = @self_modulated_batch_norm`.

* the key space of a self-modulated resnet_cifar generator against the reference's list (resnet_norm_test.py:230-306),
  the u_vars under spectral norm, the initial values, the errors and the gin binding of num_hidden;
* the kernel calls a generator forward and backward make: one modulation launch per layer forward, at most two backward;
* engine vs the oracle and its float64 twin through full training cycles (losses, every gradient, BN state, moving
  averages or accumulators), and the condition-number tangents of a self-modulated generator;
* on the H100: the three entries of csrc/modulation.cu against a float64 restatement at edge shapes, bit-identical
  reruns, network cycles in math_mode 0, graph replay == eager.

The CPU bodies run above the emulated C-ABI (tests/abi_emulator.py), with the new entries restated below."""
import contextlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import nets as onets
from tests.abi_emulator import EmulatedLib, emulated_library, f32
from tests.self_modulation_oracle import self_modulated_generators

HERE = os.path.dirname(os.path.abspath(__file__))
BINDING = "G.batch_norm_fn = @self_modulated_batch_norm"
U32 = float(np.finfo(np.float32).eps) / 2


# ------------------------------------------------------------------------------------------ float64 restatement

def ref_forward(z, wh, bh, wg, bg, wb, bb):
  """(gb [2N, C], h [N, H] or None, bound on |gb - gb64| for a fixed-order fp32 evaluation) in float64."""
  z = z.astype(np.float64)
  if wh is None:
    h, h_err = z, np.zeros_like(z)
  else:
    pre = z @ wh + bh
    h = np.maximum(pre, 0)
    h_err = (z.shape[1] + 2) * U32 * (np.abs(z) @ np.abs(wh) + np.abs(bh))
  k = h.shape[1]
  out, err = [], []
  for w, b in ((wg, bg), (wb, bb)):
    out.append(h @ w + b)
    err.append((k + 2) * U32 * (np.abs(h) @ np.abs(w) + np.abs(b)) + h_err @ np.abs(w))
  return np.concatenate(out), (None if wh is None else h), np.concatenate(err)


def ref_backward(dgb, h, z, wh, wg, wb):
  """Float64 gradients for the cotangent dgb, the fp32 h (its mask and the wide layer's input) given."""
  n = z.shape[0]
  dgb, z = dgb.astype(np.float64), z.astype(np.float64)
  dg, db = dgb[:n], dgb[n:]
  hid = z if wh is None else h.astype(np.float64)
  out = {"dw_gamma": hid.T @ dg, "db_gamma": dg.sum(0), "dw_beta": hid.T @ db, "db_beta": db.sum(0)}
  dh = dg @ wg.T + db @ wb.T
  if wh is None:
    out["dz"] = dh
  else:
    dh = dh * (h > 0)
    out.update(dw_h=z.T @ dh, db_h=dh.sum(0), dz=dh @ wh.T)
  return out


def ref_jvp(tz, h, wh, wg, wb, k):
  th = tz.astype(np.float64)
  if wh is not None:
    th = (th @ wh) * np.repeat(h > 0, k, axis=0)
  return np.concatenate([th @ wg, th @ wb])


# ------------------------------------------------------------------------------------------ emulated entries

def _arr(ptr, *shape):
  return None if ptr is None else f32(ptr, int(np.prod(shape))).reshape(shape).astype(np.float64)


def _emu_fwd(self, gb, h, z, n, zd, hidden, wh, bh, wg, bg, wb, bb, c):
  k = hidden or zd
  out, hh, _ = ref_forward(_arr(z, n, zd), _arr(wh, zd, hidden), _arr(bh, hidden), _arr(wg, k, c), _arr(bg, c),
                           _arr(wb, k, c), _arr(bb, c))
  f32(gb, 2 * n * c)[:] = out.ravel()
  if hidden:
    f32(h, n * hidden)[:] = hh.ravel()


def _emu_bwd(self, dwh, dbh, dwg, dbg, dwb, dbb, dz, dgb, h, z, wh, wg, wb, n, zd, hidden, c):
  k = hidden or zd
  g = ref_backward(_arr(dgb, 2 * n, c), _arr(h, n, hidden), _arr(z, n, zd), _arr(wh, zd, hidden), _arr(wg, k, c),
                   _arr(wb, k, c))
  for ptr, key in ((dwh, "dw_h"), (dbh, "db_h"), (dwg, "dw_gamma"), (dbg, "db_gamma"), (dwb, "dw_beta"),
                   (dbb, "db_beta"), (dz, "dz")):
    if ptr is not None:
      f32(ptr, g[key].size)[:] = g[key].ravel()


def _emu_jvp(self, tgb, tz, h, wh, wg, wb, n, zd, hidden, c, k):
  kk = hidden or zd
  out = ref_jvp(_arr(tz, n * k, zd), _arr(h, n, hidden), _arr(wh, zd, hidden), _arr(wg, kk, c), _arr(wb, kk, c), k)
  f32(tgb, out.size)[:] = out.ravel()


_EMULATED = {"cgan_self_modulation_fwd": _emu_fwd, "cgan_self_modulation_bwd": _emu_bwd,
             "cgan_self_modulation_jvp": _emu_jvp}


@pytest.fixture
def emulated(monkeypatch):
  for name, fn in _EMULATED.items():
    monkeypatch.setattr(EmulatedLib, name, fn, raising=False)
  from compare_gan_b200 import kernels as K
  with emulated_library() as lib:
    yield K, lib


@pytest.fixture(autouse=True)
def _oracle_generators():
  with self_modulated_generators():
    yield


@pytest.fixture(scope="module")
def gpu():
  from compare_gan_b200 import kernels as K
  K.init(0)
  return K


@contextlib.contextmanager
def oracle_cfg(**kw):
  """Every oracle Cfg built inside this scope gets `kw` (self_modulated = True and the generator's latent options, see
  tests/self_modulation_oracle.py) on top of what tests.gpu_util.make_pair sets."""
  base = onets.Cfg

  class Cfg(base):
    def __init__(self, **k):
      super(Cfg, self).__init__(**k)
      for name, v in kw.items():
        setattr(self, name, v)
  onets.Cfg = Cfg
  try:
    yield
  finally:
    onets.Cfg = base


def sbn_pair(arch, shape, batch, num_hidden=32, gin_extra=(), oracle_extra=None, **kw):
  """tests.gpu_util.make_pair with a self-modulated generator on both sides."""
  from tests.gpu_util import make_pair
  bindings = (BINDING, "self_modulated_batch_norm.num_hidden = %d" % num_hidden) + tuple(gin_extra)
  kw["extra_bindings"] = tuple(kw.get("extra_bindings", ())) + bindings
  with oracle_cfg(self_modulated=True, sbn_hidden=num_hidden, **(oracle_extra or {})):
    return make_pair(arch, shape, batch, **kw)


# ------------------------------------------------------------------------------------------ 1, 2, 5: names and values

def _fixture():
  with open(os.path.join(HERE, "golden", "self_modulated_variables.json")) as f:
    return json.load(f)


def test_fixture_is_the_reference_list():
  fx = _fixture()
  names = [n for n, _ in fx["variables"]]
  assert len(names) == 64 and len(set(names)) == 64
  assert names[4:10] == ["generator/B1/bn1/sbn/%s/%s:0" % (a, b) for a in ("hidden", "gamma", "beta")
                         for b in ("kernel", "bias")]


@pytest.mark.parametrize("g_sn", [False, True])
def test_key_space_initial_values_and_u_vars(emulated, g_sn):
  eng, _ = sbn_pair("resnet_cifar_arch", (32, 32, 3), 2, g_sn=g_sn)
  want = [(n[:-2], s) for n, s in _fixture()["variables"]]
  got = [(k, list(v.shape)) for k, v in eng.store.trainable.items() if k.startswith("generator/")]
  assert got == want
  state = eng.state_numpy()
  u_vars = [k for k in state if k.startswith("generator/") and "/sbn/" in k and k.endswith("/u_var")]
  kernels = [k for k, _ in want if "/sbn/" in k and k.endswith("/kernel")]
  assert sorted(u_vars) == (sorted(k + "/u_var" for k in kernels) if g_sn else [])
  for k, _ in want:
    if "/sbn/" in k and k.endswith("/bias"):
      np.testing.assert_array_equal(state[k], 1.0 if "/gamma/" in k else 0.0)
  # BN state precedes the sbn variables in each layer's scope, as in the reference
  keys = list(state)
  assert keys.index("generator/B1/bn1/moving_mean") < keys.index("generator/B1/bn1/sbn/hidden/kernel")


def test_errors_and_gin_binding(emulated):
  with pytest.raises(ValueError, match="provide z"):
    sbn_pair("resnet_cifar_arch", (32, 32, 3), 2, gin_extra=("D.batch_norm_fn = @self_modulated_batch_norm",))
  eng, _ = sbn_pair("resnet_cifar_arch", (32, 32, 3), 2, num_hidden=7)
  assert list(eng.store.trainable["generator/B1/bn1/sbn/hidden/kernel"].shape) == [128, 7]
  eng, _ = sbn_pair("resnet_cifar_arch", (32, 32, 3), 2, num_hidden=0)
  assert list(eng.store.trainable["generator/final_norm/sbn/gamma/kernel"].shape) == [128, 256]
  assert not any("/hidden/" in k for k in eng.store.trainable)


# ------------------------------------------------------------------------------------------ 3: kernel calls

def _calls(lib, fn):
  names = []
  orig = lib.call

  def call(name, *args):
    names.append(name)
    return orig(name, *args)
  lib.call = call
  try:
    fn()
  finally:
    lib.call = orig
  return names


def _count(names, *keys):
  return sum(1 for n in names if n in keys)


def test_one_launch_per_layer_forward_and_at_most_two_backward(emulated):
  K, lib = emulated
  from compare_gan_b200 import tape, variables as V
  runs = {}
  for label, bind in (("plain", False), ("sbn", True)):
    if bind:
      eng, _ = sbn_pair("resnet_cifar_arch", (32, 32, 3), 2, z_dim=16)
    else:
      from tests.gpu_util import make_pair
      eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 2, z_dim=16)
    z = K.from_numpy(np.random.RandomState(0).uniform(-1, 1, (2, 16)).astype(np.float32))
    params = [v for k, v in eng.store.trainable.items() if k.startswith("generator/")]
    with V.use(eng.store):
      out = {}

      def fwd():
        out["img"] = eng.generator(z, y=None, is_training=True)
      f = _calls(lib, fwd)
      seed = K.fill_(K.empty(*out["img"].shape), 1.0)
      b = _calls(lib, lambda: tape.backward([(out["img"], seed)], params, K.add_grad))
    runs[label] = (f, b)
  (pf, pb), (sf, sb) = runs["plain"], runs["sbn"]
  layers = 7
  assert _count(sf, "self_modulation_fwd") == layers
  for key in ("gemm", "bias_add", "act_fwd", "bn_apply", "bn_moments"):
    assert _count(sf, key) == _count(pf, key), key
  assert _count(sb, "self_modulation_bwd") == layers          # the emulator counts entries; each is <= 2 launches
  for key in ("gemm", "colsum", "act_bwd"):
    assert _count(sb, key) == _count(pb, key), key


# ------------------------------------------------------------------------------------------ 4: engine vs oracle cycles

# name: (architecture, image shape, batch, num_hidden, make_pair keywords, gin lines, oracle Cfg extras, z_dim)
CYCLES = {
    "resnet_cifar": ("resnet_cifar_arch", (32, 32, 3), 4, 32, {}, (), {}, 128),
    "resnet_cifar_hierarchical_z": ("resnet_cifar_arch", (32, 32, 3), 4, 32, {},
                                    ("resnet_cifar.Generator.hierarchical_z = True",), {"hierarchical_z": True}, 128),
    "resnet_cifar_embed_z": ("resnet_cifar_arch", (32, 32, 3), 4, 32, {},
                             ("resnet_cifar.Generator.embed_z = True",), {"embed_z": True}, 128),
    "resnet_cifar_hidden0": ("resnet_cifar_arch", (32, 32, 3), 4, 0, {}, (), {}, 128),
    "resnet_cifar_sn": ("resnet_cifar_arch", (32, 32, 3), 4, 32, {"g_sn": True, "d_sn": True}, (), {}, 128),
    "resnet_cifar_accumulators": ("resnet_cifar_arch", (32, 32, 3), 4, 32, {"use_moving_averages": False}, (), {}, 128),
    "resnet5": ("resnet5_arch", (64, 64, 3), 2, 32, {}, (), {}, 128),
    "sndcgan": ("sndcgan_arch", (32, 32, 3), 4, 32, {}, (), {}, 128),
    "dcgan": ("dcgan_arch", (32, 32, 3), 4, 32, {}, (), {}, 128),
    "biggan": ("resnet_biggan_arch", (32, 32, 3), 4, 32, {"ch": 8, "conditional": True, "num_classes": 10}, (), {}, 120),
    "biggan_deep": ("resnet_biggan_deep_arch", (32, 32, 3), 2, 16, {"ch": 4, "conditional": True, "num_classes": 10}, (),
                    {}, 128),
}


# BigGAN (D gradients of order 1e-7 in its last blocks) and sndcgan at 128x128 (g_bn1 normalises each of its 131,072
# channels over 4 samples) amplify Adam's sign noise past the generic post-update bounds: they are checked with D frozen
FROZEN_D_ONLY = ("biggan", "biggan_deep", "sndcgan_128")


def check_cycle(name, math_mode=0, cycles=True):
  """One cycle with D frozen (tight G gradients against float64, sbn ones included), then (`cycles`) two ordinary
  cycles: losses, gradients, weights after Adam and BN state (tests/test_gan_step_gpu.py's criteria)."""
  import tests.test_gan_step_gpu as steps
  arch, shape, batch, hidden, kw, gin_extra, oextra, zd = CYCLES[name]
  from tests import gpu_util
  orig = gpu_util.make_pair

  def make_pair(arch, image_shape, batch, **k):
    return sbn_pair(arch, image_shape, batch, num_hidden=hidden, gin_extra=gin_extra, oracle_extra=oextra, **k)
  steps.make_pair = make_pair
  try:
    worst = steps._frozen_d_gradients(batch, shape, zd, 1, arch=arch, math_mode=math_mode,
                                      **{k: v for k, v in kw.items() if k != "num_classes"},
                                      num_classes=kw.get("num_classes", 0))
    eng, orc = make_pair(arch, shape, batch, z_dim=zd, disc_iters=2, math_mode=math_mode, **kw)
    assert any("/sbn/" in k for k in eng.flat_g["views"])
    if cycles:
        steps._cycles_both(eng, orc, batch, shape, zd, 2, num_classes=kw.get("num_classes", 0))
  finally:
    steps.make_pair = orig
  return eng, orc, worst


@pytest.mark.parametrize("name", ["resnet_cifar", "resnet_cifar_hierarchical_z", "resnet_cifar_embed_z",
                                  "resnet_cifar_hidden0", "resnet_cifar_sn", "resnet_cifar_accumulators", "sndcgan",
                                  "dcgan", "biggan", "biggan_deep"])
def test_cycles_match_the_oracle_on_the_emulator(emulated, name):
  check_cycle(name, cycles=name not in FROZEN_D_ONLY)


@pytest.mark.parametrize("hidden", [32, 0])
def test_condition_number_tangents_on_the_emulator(emulated, monkeypatch, hidden):
  import tests.test_jacobian_conditioning as jc
  monkeypatch.setattr(jc, "_EMULATED", dict(jc._EMULATED))
  for name, fn in jc._EMULATED.items():
    monkeypatch.setattr(EmulatedLib, name, fn, raising=False)
  K, _ = emulated
  monkeypatch.setitem(jc.GENERATORS, "resnet_cifar_sbn", (
      "resnet_cifar_arch", (32, 32, 3),
      dict(extra_bindings=(BINDING, "self_modulated_batch_norm.num_hidden = %d" % hidden)), 8))
  with oracle_cfg(self_modulated=True, sbn_hidden=hidden):
    jc.check_generator(K, "resnet_cifar_sbn")


# ------------------------------------------------------------------------------------------ 7-9: on the H100

def _draw(rs, n, zd, hidden, c):
  k = hidden or zd
  z = rs.uniform(-1, 1, (n, zd)).astype(np.float32)
  wh = (rs.standard_normal((zd, hidden)) * 0.3).astype(np.float32) if hidden else None
  bh = (rs.standard_normal(hidden) * 0.1).astype(np.float32) if hidden else None
  wg, wb = [(rs.standard_normal((k, c)) * 0.1).astype(np.float32) for _ in range(2)]
  bg, bb = (1 + 0.1 * rs.standard_normal(c)).astype(np.float32), (0.1 * rs.standard_normal(c)).astype(np.float32)
  return z, wh, bh, wg, bg, wb, bb


def _bound_check(got, want, bound, what):
  bad = np.abs(got.astype(np.float64) - want) > bound + 1e-30
  assert not bad.any(), "%s: %d elements outside the fp32 bound, worst %.3e vs %.3e" % (
      what, int(bad.sum()), float(np.abs(got - want).max()), float(bound.max()))


ENTRY_SHAPES = [(n, zd, hidden, c) for n, zd, hidden in
                [(1, 20, 32), (7, 32, 0), (64, 128, 32), (256, 128, 100), (64, 20, 100), (7, 128, 0), (256, 32, 0),
                 (1, 128, 100)]
                for c in (3, 200, 256, 1536, 8192)] + [(64, 128, 32, 131072), (7, 20, 0, 131072), (256, 32, 100, 131072)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,zd,hidden,c", ENTRY_SHAPES)
def test_entries_match_float64(gpu, n, zd, hidden, c):
  K = gpu
  rs = np.random.RandomState(n * 7 + zd + hidden + c % 997)
  z, wh, bh, wg, bg, wb, bb = _draw(rs, n, zd, hidden, c)
  dev = lambda a: None if a is None else K.from_numpy(a)
  Z, WH, BH, WG, BG, WB, BB = [dev(a) for a in (z, wh, bh, wg, bg, wb, bb)]
  k = hidden or zd

  def fwd():
    gb, h = K.empty(2 * n, c), (K.empty(n, hidden) if hidden else None)
    K._call("self_modulation_fwd", gb.ptr, None if h is None else h.ptr, Z.ptr, n, zd, hidden,
            None if WH is None else WH.ptr, None if BH is None else BH.ptr, WG.ptr, BG.ptr, WB.ptr, BB.ptr, c)
    return gb.cpu(), (None if h is None else h.cpu())
  gb, h = fwd()
  gb2, h2 = fwd()
  np.testing.assert_array_equal(gb, gb2)
  want, h64, bound = ref_forward(z, wh, bh, wg, bg, wb, bb)
  _bound_check(gb, want, bound, "gb")
  if hidden:
    np.testing.assert_array_equal(h2, h)
    hb = (zd + 2) * U32 * (np.abs(z.astype(np.float64)) @ np.abs(wh) + np.abs(bh))
    _bound_check(h, h64, hb, "h")

  dgb = rs.standard_normal((2 * n, c)).astype(np.float32)
  DGB, H = K.from_numpy(dgb), (K.from_numpy(h) if hidden else None)

  def bwd():
    outs = {"dw_gamma": K.empty(k, c), "db_gamma": K.empty(c), "dw_beta": K.empty(k, c), "db_beta": K.empty(c),
            "dz": K.empty(n, zd)}
    if hidden:
      outs.update(dw_h=K.empty(zd, hidden), db_h=K.empty(hidden))
    p = lambda key: outs[key].ptr if key in outs else None
    K._call("self_modulation_bwd", p("dw_h"), p("db_h"), p("dw_gamma"), p("db_gamma"), p("dw_beta"), p("db_beta"),
            p("dz"), DGB.ptr, None if H is None else H.ptr, Z.ptr, None if WH is None else WH.ptr, WG.ptr, WB.ptr, n, zd,
            hidden, c)
    return {key: v.cpu() for key, v in outs.items()}
  g1, g2 = bwd(), bwd()
  ref = ref_backward(dgb, h, z, wh, wg, wb)
  a = np.abs
  hid = a(z.astype(np.float64)) if not hidden else a(h.astype(np.float64))
  dg, db = a(dgb[:n].astype(np.float64)), a(dgb[n:].astype(np.float64))
  dh_scale = dg @ a(wg).T + db @ a(wb).T
  dh_bound = (2 * c + 2) * U32 * dh_scale
  bounds = {"dw_gamma": (n + 2) * U32 * (hid.T @ dg), "db_gamma": (n + 2) * U32 * dg.sum(0),
            "dw_beta": (n + 2) * U32 * (hid.T @ db), "db_beta": (n + 2) * U32 * db.sum(0)}
  if hidden:
    m = h > 0
    bounds.update(dw_h=(n + 2) * U32 * (a(z).T @ (dh_scale * m)) + a(z).T @ (dh_bound * m),
                  db_h=(n + 2) * U32 * (dh_scale * m).sum(0) + (dh_bound * m).sum(0),
                  dz=(hidden + 2) * U32 * ((dh_scale * m) @ a(wh).T) + (dh_bound * m) @ a(wh).T)
  else:
    bounds["dz"] = dh_bound
  for key in g1:
    np.testing.assert_array_equal(g1[key], g2[key])
    _bound_check(g1[key], ref[key], bounds[key], key)

  kt = 3
  tz = rs.standard_normal((n * kt, zd)).astype(np.float32)
  TGB = K.empty(2 * n * kt, c)
  K._call("self_modulation_jvp", TGB.ptr, K.from_numpy(tz).ptr, None if H is None else H.ptr,
          None if WH is None else WH.ptr, WG.ptr, WB.ptr, n, zd, hidden, c, kt)
  tw = ref_jvp(tz, h, wh, wg, wb, kt)
  th = a(tz.astype(np.float64))
  if hidden:
    m = np.repeat(h > 0, kt, axis=0)
    th_b = (zd + 2) * U32 * (th @ a(wh)) * m
    th = (th @ a(wh)) * m
  else:
    th_b = np.zeros_like(th)
  tb = np.concatenate([(k + 2) * U32 * (th @ a(w)) + th_b @ a(w) for w in (wg, wb)])
  _bound_check(TGB.cpu(), tw, tb, "t_gb")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["resnet_cifar", "resnet_cifar_embed_z", "resnet_cifar_hidden0", "sndcgan", "biggan"])
def test_cycles_match_the_oracle(gpu, name):
  check_cycle(name, cycles=name not in FROZEN_D_ONLY)


@pytest.mark.gpu
def test_sndcgan_128_cycle_matches_the_oracle(gpu, monkeypatch):
  monkeypatch.setitem(CYCLES, "sndcgan_128", ("sndcgan_arch", (128, 128, 3), 4, 32, {}, (), {}, 128))
  check_cycle("sndcgan_128", cycles=False)


@pytest.mark.gpu
def test_graph_replay_equals_eager(gpu):
  from tests.gpu_util import make_inputs
  eng, _ = sbn_pair("resnet_cifar_arch", (32, 32, 3), 4, disc_iters=2)
  rng = np.random.RandomState(9)
  batches = [make_inputs(rng, 2, 4, (32, 32, 3), 128) for _ in range(2)]
  snap = eng.snapshot()
  eager = []
  for b in batches:
    eng.set_inputs(*b)
    eng.run_cycle()
    eager.append(eng.read_losses())
  state_eager = eng.state_numpy()
  eng.restore(snap)
  eng.capture(warmup=2)
  for i, b in enumerate(batches):
    eng.set_inputs(*b)
    eng.run_cycle()
    assert eng.read_losses() == eager[i]
  for k, v in eng.state_numpy().items():
    np.testing.assert_array_equal(v, state_eager[k], err_msg=k)
