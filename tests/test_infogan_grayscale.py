"""The infogan architecture, the MNIST / Fashion-MNIST data sets, and the tensor-core routes that 28x28x1 networks need:
stride-2 input gradients (every transposed convolution) and filter gradients over odd grids, and the stride-2 input
gradient of image-side layers (dx with <= 4 channels).

CPU: both data sets through get_dataset (shapes, labels, the fake set, shard naming, errors), the infogan variables
against tests/golden/infogan_grayscale.json and the float64-capable restatement in tests/infogan_oracle.py, and the
engine against that restatement above the emulated C-ABI (forward passes and full cycles at five image shapes, dcgan and
sndcgan at 28x28x1 and 32x32x1).
GPU: every new route element by element against float64 (tests/test_tc_exact_gpu.py's criterion), pixels past a phase's
extent left untouched, old routes with their old bits; infogan and sndcgan at 28x28x1 in math_mode 0 and 1, with every
convolution call on the tensor cores in math_mode 1; CUDA-graph replay; run_with_schedule on mnist."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import nets as onets
from tests import arch_trace as at
from tests import infogan_oracle  # noqa: F401  (adds the pair to the oracle's tables)
from tests.abi_emulator import emulated_library
from tests.gpu_util import make_inputs, make_pair

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_PATH = os.path.join(HERE, "golden", "infogan_grayscale.json")
INFOGAN = "infogan_arch"
GRAY28 = (28, 28, 1)


def golden():
  return json.load(open(GOLDEN_PATH))


# ------------------------------------------------------------------------------------------ data sets (CPU)

@pytest.mark.parametrize("key,name", [("mnist", "mnist"), ("fashion-mnist", "fashion_mnist")])
def test_grayscale_datasets(key, name, tmp_path):
  from compare_gan_b200 import datasets
  ds = datasets.get_dataset(key)
  assert ds.name == name and ds.image_shape == GRAY28 and ds.num_classes == 10 and ds.eval_test_samples == 10000
  assert ds.sample_images(3).shape == (3, 28, 28, 1) and ds.sample_labels(3).max() < 10
  it = ds.train_input_fn(params={"batch_size": 8})
  images, labels = next(it)
  assert images.shape == (8, 28, 28, 1) and images.dtype == np.float32 and (labels == 1).all()     # the fake set
  assert 0.0 <= images.min() and images.max() < 1.0
  it.close()
  # uint8 shards named after the data set (not the key), read through the native loader
  rng = np.random.RandomState(0)
  shards = {}
  for split in ("train", "test"):
    shards[split] = rng.randint(0, 256, (16, 28, 28, 1)).astype(np.uint8)
    np.save(str(tmp_path / ("%s_%s_images.npy" % (name, split))), shards[split])
    np.save(str(tmp_path / ("%s_%s_labels.npy" % (name, split))), np.arange(16) % 10)
  real = datasets.get_dataset(key, fake_dataset=False, data_dir=str(tmp_path))
  it = real.eval_input_fn(params={"batch_size": 8})
  batches = list(it)
  assert len(batches) == 2
  np.testing.assert_array_equal(batches[0][0], shards["test"][:8].astype(np.float32) / 255.0)
  np.testing.assert_array_equal(batches[1][1], np.arange(8, 16) % 10)
  it.close()
  # errors: no data_dir, shards of the wrong geometry, and the key spelled as the name
  with pytest.raises(ValueError, match="no data_dir"):
    datasets.get_dataset(key, fake_dataset=False, data_dir="").train_input_fn(params={"batch_size": 8})
  np.save(str(tmp_path / ("%s_train_images.npy" % name)), np.zeros((4, 32, 32, 1), np.uint8))
  with pytest.raises(ValueError, match=r"uint8 \[N,28,28,1\]"):
    real.train_input_fn(params={"batch_size": 2})
  if key != name:
    with pytest.raises(ValueError, match="not available"):
      datasets.get_dataset(name)


# ------------------------------------------------------------------------------------------ definitions (CPU)

def _counts(variables):
  g = sum(int(np.prod(s)) for n, s, t in variables if t and n.startswith("generator/"))
  d = sum(int(np.prod(s)) for n, s, t in variables if t and n.startswith("discriminator/"))
  return g, d


def _oracle_variables(image_shape, z_dim, d_bn=None, d_sn=False):
  import torch
  cfg = onets.Cfg(architecture=INFOGAN, image_shape=image_shape, d_bn=d_bn, d_sn=d_sn)
  store = onets.VarStore()
  with torch.no_grad():
    img = onets.generator(store, cfg, torch.zeros(2, z_dim), None, True)
    onets.discriminator(store, cfg, img, None, True)
  return [[k, list(v.shape), k in store.trainable] for k, v in store.vars.items()]


# (gin bindings, image shape, z_dim) of the pinned variable lists; G.batch_norm_fn is bound to show that it does not
# reach infogan's generator
VARIABLE_CASES = {
    "mnist": ("G.batch_norm_fn = None", GRAY28, 64),
    "mnist_d_bn_sn": ("G.batch_norm_fn = @conditional_batch_norm\nD.batch_norm_fn = @batch_norm\nD.spectral_norm = True\n"
                      "D.layer_norm = True", GRAY28, 64),
    "rgb_64": ("G.batch_norm_fn = @batch_norm", (64, 64, 3), 128),
}


def write_golden(path=GOLDEN_PATH, old_route_bits=None):
  """Regenerates the variable lists from the CURRENT definitions (only after an intended change); `old_route_bits`
  (sha1 per OLD_ROUTE_CASES id, measured on an H100 with the library before the new routes) is kept if not given."""
  g = {"_about": "infogan variables (name, shape, trainable) and trainable counts per configuration of "
                 "tests/test_infogan_grayscale.py:VARIABLE_CASES; old_route_bits: sha1 of the float32 result of each "
                 "OLD_ROUTE_CASES contraction as computed before the odd-grid and image-side stride-2 routes existed."}
  for name, (gin_text, shape, z_dim) in VARIABLE_CASES.items():
    v = [x[:3] for x in at.trace_networks(gin_text, INFOGAN, shape, z_dim=z_dim)["variables"]]
    g[name] = {"variables": v, "trainable_g": _counts(v)[0], "trainable_d": _counts(v)[1]}
  old = json.load(open(path)).get("old_route_bits") if os.path.exists(path) else None
  g["old_route_bits"] = old_route_bits or old or {}
  json.dump(g, open(path, "w"), indent=0)


def test_parameter_counts_at_28x28x1():
  """Counted by hand from the reference's definitions: G 6,642,241, D 6,556,865 at z_dim 64 without D normaliser or SN."""
  v = [x[:3] for x in at.trace_networks("G.batch_norm_fn = None", INFOGAN, GRAY28, z_dim=64)["variables"]]
  assert _counts(v) == (6642241, 6556865)


@pytest.mark.parametrize("case", sorted(VARIABLE_CASES))
def test_variables_match_the_golden_and_the_restatement(case):
  gin_text, shape, z_dim = VARIABLE_CASES[case]
  want = golden()[case]
  v = [x[:3] for x in at.trace_networks(gin_text, INFOGAN, shape, z_dim=z_dim)["variables"]]
  assert v == want["variables"]
  assert _counts(v) == (want["trainable_g"], want["trainable_d"])
  d_bn = "batch_norm" if "D.batch_norm_fn" in gin_text else None
  assert v == _oracle_variables(shape, z_dim, d_bn=d_bn, d_sn="D.spectral_norm = True" in gin_text)
  names = [x[0] for x in v]
  assert "generator/g_bn1/gamma" in names and not any("condition" in n for n in names)     # plain BN in G regardless
  assert ("discriminator/d_bn2/gamma" in names) == (d_bn is not None)


# ------------------------------------------------------------------------------------------ networks vs the restatement

def _net(arch, shape, batch=4, z_dim=64, k=1, **kw):
  from tests.test_gan_step_gpu import _cycles_both, _forward_both
  eng, orc = make_pair(arch, shape, batch, disc_iters=k, z_dim=z_dim, **kw)
  _forward_both(eng, orc, batch, z_dim)          # G's images and D's probabilities in [0, 1] (architectures_test.py)
  _cycles_both(eng, orc, batch, shape, z_dim, k)


def _infogan_d_bn(shape):
  """D.batch_norm_fn = @batch_norm on both sides (make_pair binds G's normaliser only)."""
  import functools
  from unittest import mock
  with mock.patch.object(onets, "Cfg", functools.partial(onets.Cfg, d_bn="batch_norm")):
    _net(INFOGAN, shape, d_sn=True, extra_bindings=["D.batch_norm_fn = @batch_norm"])


NETWORK_CASES = {
    "infogan_28x28x1": lambda: _net(INFOGAN, GRAY28, k=2),
    "infogan_28x28x1_d_bn_sn": lambda: _infogan_d_bn(GRAY28),
    "infogan_32x32x1": lambda: _net(INFOGAN, (32, 32, 1), d_sn=True),
    "infogan_32x32x3": lambda: _net(INFOGAN, (32, 32, 3)),
    "infogan_64x64x3": lambda: _net(INFOGAN, (64, 64, 3), batch=2, z_dim=128, d_sn=True),
    "infogan_128x128x3": lambda: _net(INFOGAN, (128, 128, 3), batch=2, z_dim=128),
    "dcgan_28x28x1": lambda: _net("dcgan_arch", GRAY28, z_dim=128),
    "dcgan_32x32x1": lambda: _net("dcgan_arch", (32, 32, 1), z_dim=128),
    "sndcgan_28x28x1": lambda: _net("sndcgan_arch", GRAY28, d_sn=True),
    "sndcgan_32x32x1": lambda: _net("sndcgan_arch", (32, 32, 1), d_sn=True),
}


@pytest.mark.parametrize("case", sorted(NETWORK_CASES))
def test_networks_match_the_restatement_on_the_emulator(case):
  with emulated_library() as lib:
    NETWORK_CASES[case]()
    assert lib.launches > 0


# ------------------------------------------------------------------------------------------ kernels (GPU)

def _route_cases():
  from tests.test_tc_exact_gpu import dgrad, wgrad
  cases = []
  # (1) stride-2 input gradients through the output phases: odd and even sides, 3x3 and 4x4 (5x5 stays on its old path)
  for i, (h, w) in enumerate([(3, 5), (7, 7), (9, 15), (17, 29), (15, 4), (29, 17), (5, 9), (4, 7)]):
    k = (3, 4)[i % 2]
    ep = [dict(bias=True), dict(residual=True), dict(leak=0.2), dict(bias=True, residual=True), dict(leak=0.0),
          dict(bias=True, leak=0.2), {}, dict(bias=True)][i]
    cin, cout = [(32, 64), (64, 32), (128, 64), (64, 96), (32, 32), (64, 64), (256, 128), (48, 64)][i]
    cases.append(dgrad("dgrad s2 odd", 2, h, w, cin, cout, k, k, stride=2, launches=2, **ep))
  # the layers of sndcgan at 28x28: g_dc2 (4 -> 7) and d_conv6 (7 -> 4)
  cases.append(dgrad("dgrad s2 odd", 4, 7, 7, 256, 512, 4, 4, stride=2, bias=True, launches=2, note="sndcgan28"))
  cases.append(dgrad("dgrad s2 odd", 4, 7, 7, 256, 512, 4, 4, stride=2, leak=0.1, launches=2, note="sndcgan28-mask"))
  # (2) stride-2 filter gradients over odd grids, 3x3 and 4x4 (the wgmma filter-gradient kernel takes at most 16 taps;
  # batches for which its box rule tiles the dY grid: a 2-wide grid needs a multiple of 8 images, a 2 x 4 one of 4)
  for i, (n, h, w) in enumerate([(8, 3, 3), (2, 7, 5), (2, 7, 7), (2, 9, 5), (2, 15, 17), (2, 17, 13), (2, 29, 29),
                                 (4, 7, 4)]):
    k = (3, 4)[i % 2]
    cases.append(wgrad("wgrad s2 odd", n, h, w, (64, 96, 128)[i % 3], (64, 32, 96)[i % 3], k, k, stride=2))
  cases.append(wgrad("wgrad s2 odd", 4, 7, 7, 256, 512, 4, 4, stride=2, note="sndcgan28"))
  # (3) image-side stride-2 input gradients, kh kw cin <= 32: infogan's g_dc4 / d_conv1 (cin 1) and the other widths
  # (cin 4: a 2x2 kernel stays with the phase kernel of route (1), a 3x1 one has empty phases and takes this route)
  for cin, (kh, kw), (h, w), ep in [(1, (4, 4), (28, 28), dict(bias=True)), (1, (5, 5), (9, 7), {}),
                                    (2, (4, 4), (15, 16), dict(leak=0.2)), (2, (3, 3), (7, 9), dict(bias=True, residual=True)),
                                    (3, (3, 3), (17, 17), dict(bias=True)), (3, (3, 3), (8, 12), {}),
                                    (4, (2, 2), (9, 5), dict(bias=True)), (4, (3, 1), (11, 6), dict(bias=True, leak=0.2)),
                                    (1, (3, 3), (3, 3), {})]:
    cases.append(dgrad("dgrad s2 thin-cin", 2, h, w, cin, 64, kh, kw, stride=2, **ep))
  cases.append(dgrad("dgrad s2 thin-cin", 4, 28, 28, 1, 64, 4, 4, stride=2, leak=0.2, note="infogan28"))
  return cases


ROUTE_IDS = [c.id for c in _route_cases()]


@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  kernels.set_math_mode(1)
  yield kernels
  kernels.set_math_mode(0)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(ROUTE_IDS)), ids=ROUTE_IDS)
def test_new_routes_elementwise(K, i):
  from tests import test_tc_exact_gpu as tce
  tce.check_case(K, _route_cases()[i])


def _run_into_guarded(K, c, a, b, ex, sentinel=np.float32(-1234.5)):
  """The case's call writing into the front of a sentinel-filled buffer one image longer than its output; returns
  (output, tail)."""
  from compare_gan_b200 import _lib
  from tests import test_tc_exact_gpu as tce
  shape = tce.out_shape(c)
  size = int(np.prod(shape))
  buf = K.from_numpy(np.full(size + size // shape[0], sentinel, np.float32))
  A, B = K.from_numpy(a), K.from_numpy(b)
  dev = {k: K.from_numpy(v) for k, v in ex.items()}
  ep = K._epilogue(dev.get("bias"), dev.get("residual"), dev.get("mask"), c.leak or 0.0, c.relu, False, False)
  K._call("conv2d_dgrad_ex", ctypes.byref(tce.desc(K, c)), A.ptr, B.ptr, ctypes.byref(ep), buf.ptr)
  assert _lib.PATH_NAMES[K.lib().get_option(_lib.OPT_LAST_PATH)] == "tcgen05_tf32"
  out = np.array(buf.cpu(), copy=True)
  return out[:size].reshape(shape), out[size:]


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(7, 7), (9, 4), (4, 9), (15, 17)])
def test_pixels_past_a_phase_extent_stay_untouched(K, h, w):
  """An odd dx has odd phases one row / column short: the image after it (and, for the last image, the memory after
  the tensor) keeps its sentinel, with the register epilogue and with the residual / mask prefetched by TMA."""
  from tests import test_tc_exact_gpu as tce
  sentinel = np.float32(-1234.5)
  for ep in (dict(bias=True), dict(residual=True), dict(leak=0.2)):
    for n in (1, 3):
      c = tce.dgrad("dgrad s2 odd", n, h, w, 64, 64, 4, 4, stride=2, **ep)
      a, b, ex = tce.draw(c)
      y64, scale = tce.reference(c, a, b, ex)
      y, tail = _run_into_guarded(K, c, a, b, ex, sentinel)
      tce.check(y, y64, scale, c.id)
      assert (tail.view(np.uint32) == sentinel.view(np.uint32)).all(), "%s: stored past dx" % c.id


def _old_route_cases():
  from tests.test_tc_exact_gpu import dgrad, fwd, wgrad
  return [
      dgrad("dgrad s2 phases", 2, 12, 16, 32, 64, 4, 4, stride=2, bias=True),
      dgrad("dgrad s2 phases", 4, 28, 28, 64, 128, 4, 4, stride=2, leak=0.1),      # sndcgan28 d_conv2
      wgrad("wgrad s2", 4, 28, 28, 64, 128, 4, 4, stride=2),
      wgrad("wgrad s2", 2, 16, 32, 64, 64, 4, 4, stride=2),
      dgrad("dgrad thin-cin", 2, 12, 20, 3, 32, 3, 3, bias=True),
      dgrad("dgrad thin-cin", 4, 28, 28, 1, 64, 3, 3, leak=0.1),                   # sndcgan28 d_conv1
      fwd("fwd thin-cout", 2, 12, 20, 64, 3, 3, 3, bias=True),
      fwd("fwd thin-cout", 4, 28, 28, 64, 1, 3, 3, bias=True),                     # sndcgan28 g_dc5
  ]


def old_route_bits(K):
  """{case id: sha1 of the float32 result} of the old-route cases with the library loaded in K (math_mode 1).  The masks
  are drawn as when the bits were recorded: without exact zeros, where the (leaky-)ReLU gate's rule at 0 does not
  enter, so the bits depend on the route alone."""
  from tests import test_tc_exact_gpu as tce
  out = {}
  for c in _old_route_cases():
    a, b, ex = tce.draw(c, mask_zeros=False)
    y, _, path = tce.run(K, c, a, b, ex)
    out[c.id] = (path, hashlib.sha1(np.ascontiguousarray(y).view(np.uint32).tobytes()).hexdigest())
  return out


@pytest.mark.gpu
def test_old_routes_keep_their_path_and_bits(K):
  """An even-size stride-2 input and filter gradient and the stride-1 image-side layers take the path they took before
  the new routes, with the same bits."""
  want = golden()["old_route_bits"]
  got = old_route_bits(K)
  assert sorted(got) == sorted(want)
  for k, (path, sha) in got.items():
    assert path == "tcgen05_tf32", (k, path)
    assert sha == want[k][1], "%s: result bits changed" % k


# ------------------------------------------------------------------------------------------ networks (GPU)

@pytest.mark.gpu
@pytest.mark.parametrize("case", ["infogan_28x28x1", "infogan_28x28x1_d_bn_sn", "sndcgan_28x28x1"])
def test_networks_match_the_restatement(case):
  NETWORK_CASES[case]()


TF32_CASES = {
    "infogan_28": dict(arch=INFOGAN, image=GRAY28, batch=8, z_dim=64, k=1, pair=dict(d_sn=True)),
    "sndcgan_28": dict(arch="sndcgan_arch", image=GRAY28, batch=16, z_dim=128, k=1, pair=dict(d_sn=True)),
}


@pytest.mark.gpu
def test_tf32_sndcgan_matches_the_oracle(monkeypatch):
  """tests/test_tf32_parity_gpu.py's check: forward activations against a TF32-emulating oracle, every contraction of a
  cycle recomputed in situ, gradients against float64."""
  import tests.test_tf32_parity_gpu as tf32_tests
  monkeypatch.setitem(tf32_tests.ARCHS, "sndcgan_28", TF32_CASES["sndcgan_28"])
  tf32_tests.test_tf32_network_parity("sndcgan_28")


@pytest.mark.gpu
def test_tf32_infogan_matches_the_oracle():
  """The bounds of tests/test_tf32_parity_gpu.py for infogan, whose forward pass has four convolutions (that check asks
  for six distinct tensor-core shapes): every observed activation within 2x of what the TF32-emulating oracle loses
  against the fp32 oracle and under the depth-scaled cap; one cycle with D frozen, every contraction recomputed in situ,
  losses, and each gradient within 3x the TF32-emulating oracle's distance to float64."""
  import torch
  from compare_gan_b200 import kernels as K, tape, variables as V
  from oracle import tf_ops as T
  from tests import test_tf32_parity_gpu as tp
  from tests.gpu_util import ReluSigns, rel_err
  c = TF32_CASES["infogan_28"]
  b, zd = c["batch"], c["z_dim"]
  eng, orc, orc64 = make_pair(INFOGAN, GRAY28, b, disc_iters=1, z_dim=zd, d_lr=1e-30, math_mode=1, with64=True, **c["pair"])
  try:
    state0 = eng.state_numpy()
    z = np.random.RandomState(31).uniform(-1, 1, (b, zd)).astype(np.float32)
    snap = eng.snapshot()
    K.CONV_TRACE = {}
    with tp._Acts() as acts:
      with V.use(eng.store), tape.no_record():
        eng.discriminator(eng.generator(K.from_numpy(z), y=None, is_training=True), y=None, is_training=True)
      plan = dict(K.CONV_TRACE)
      assert sum(1 for v in plan.values() if v[0] == "tcgen05_tf32") == 4, plan

      def oracle_forward():
        orc.store.load_numpy(state0)
        with torch.no_grad():
          onets.discriminator(orc.store, orc.cfg, onets.generator(orc.store, orc.cfg, torch.from_numpy(z), None, True),
                              None, True)
      oracle_forward()
      fp32_obs = acts.take_oracle()
      T.TF32_PLAN = plan
      try:
        oracle_forward()
      finally:
        T.TF32_PLAN = None
      emu_obs = acts.take_oracle()
    assert len(acts.eng) >= 8
    for (name, depth, te, t32), (_, _, _, temu) in zip(tp._match(acts.eng, fp32_obs), tp._match(acts.eng, emu_obs)):
      e_eng, e_emu = rel_err(te, t32), rel_err(temu, t32)
      assert e_eng <= 2.0 * e_emu + 1e-4, "%s is %.2e from fp32, the TF32-emulating oracle only %.2e" % (name, e_eng, e_emu)
      cap = max(1e-3, 4e-4 * np.sqrt(depth + 1)) if te.ndim == 4 else 5e-3
      assert e_eng <= cap, "%s is %.2e from the fp32 oracle (cap %.1e)" % (name, e_eng, cap)
    eng.restore(snap)
    orc.store.load_numpy(state0)
    orc64.store.load_numpy(state0)
    inputs = make_inputs(np.random.RandomState(37), 1, b, GRAY28, zd)
    eng.set_inputs(*inputs)
    K.CONV_TRACE = {}
    checker = tp._InSitu(K)
    K.CONV_CHECK = checker
    with ReluSigns():
      eng.run_cycle()
      dl, gl = eng.read_losses()
      K.CONV_CHECK = None
      T.TF32_PLAN = dict(K.CONV_TRACE)
      try:
        orc.cycle(*inputs)
      finally:
        T.TF32_PLAN = None
      odl, ogl = orc64.cycle(*inputs)
    assert len([r for r in checker.results if r[2] == "tcgen05_tf32"]) >= 12
    bad = [r for r in checker.results if r[0] > (2e-4 if r[2] == "tcgen05_tf32" else 3e-5) and r[3] > 1e-12]
    assert not bad, sorted(bad, reverse=True)[:5]
    assert abs(gl - ogl) <= 1e-3 * max(1.0, abs(ogl)), (gl, ogl)
    assert all(abs(a - o) <= 1e-3 * max(1.0, abs(o)) for a, o in zip(dl, odl)), (dl, odl)
    for flat, ref64, emu in ((eng.flat_d, orc64.last_d_grads, orc.last_d_grads), (eng.flat_g, orc64.last_g_grads,
                                                                                  orc.last_g_grads)):
      g = flat["grad"].cpu()
      gmax = max(float(v.norm()) for v in ref64.values())
      for name, (off, n) in flat["views"].items():
        a, r64, re = g[off:off + n].astype(np.float64), ref64[name].numpy().ravel(), emu[name].numpy().ravel().astype(np.float64)
        err, err_emu = np.linalg.norm(a - r64), np.linalg.norm(re - r64)
        bound = 3.0 * err_emu + (5e-3 if n <= 4 else 2e-3) * np.linalg.norm(r64) + 1e-5 * gmax
        assert err <= bound, "%s grad: |engine - fp64| %.3e > %.3e (|TF32-emulating oracle - fp64| %.3e)" % (
            name, err, bound, err_emu)
  finally:
    K.CONV_TRACE = None
    K.CONV_CHECK = None
    K.set_math_mode(0)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(TF32_CASES))
def test_every_convolution_of_a_cycle_runs_on_the_tensor_cores(monkeypatch, case):
  from compare_gan_b200 import _lib
  from compare_gan_b200 import kernels as K
  c = TF32_CASES[case]
  eng, _ = make_pair(c["arch"], c["image"], c["batch"], disc_iters=c["k"], z_dim=c["z_dim"], math_mode=1, **c["pair"])
  calls = []
  real_call = K._call

  def recording_call(name, *args):
    real_call(name, *args)
    if name.startswith("conv2d_"):
      desc = args[0]._obj
      calls.append((name, (desc.n, desc.h, desc.w, desc.cin, desc.cout, desc.kh, desc.stride),
                    _lib.PATH_NAMES[K.lib().get_option(_lib.OPT_LAST_PATH)]))
  monkeypatch.setattr(K, "_call", recording_call)
  try:
    eng.set_inputs(*make_inputs(np.random.RandomState(3), c["k"], c["batch"], c["image"], c["z_dim"]))
    eng.run_cycle()
    eng.read_losses()
  finally:
    K.set_math_mode(0)
  kinds = set(n for n, _, _ in calls)
  assert {"conv2d_fwd_ex", "conv2d_dgrad_ex", "conv2d_wgrad_ex"} <= kinds, kinds
  off = [x for x in calls if x[2] != "tcgen05_tf32"]
  assert not off, "calls off the tensor cores: %s" % off


@pytest.mark.gpu
@pytest.mark.parametrize("arch", [INFOGAN, "sndcgan_arch"])
def test_cuda_graph_replay_equals_eager(arch):
  from compare_gan_b200 import kernels as K
  eng, _ = make_pair(arch, GRAY28, 8, d_sn=True, disc_iters=2, z_dim=64, math_mode=1)
  try:
    rng = np.random.RandomState(9)
    batches = [make_inputs(rng, 2, 8, GRAY28, 64) for _ in range(2)]
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
      assert eng.read_losses() == eager[i], "graph replay must be bit-identical to eager"
    for k, v in eng.state_numpy().items():
      np.testing.assert_array_equal(v, state_eager[k], err_msg=k)
  finally:
    K.set_math_mode(0)


@pytest.mark.gpu
def test_run_with_schedule_on_mnist_trains_and_evaluates(tmp_path):
  """infogan on the fake mnist set: training, a checkpoint, and FID / IS of 28x28x1 samples (tiled to three channels
  for Inception) in scores.csv."""
  import csv
  from compare_gan_b200 import gin_lite as gin, runner_lib
  from compare_gan_b200.gans import modular_gan  # noqa: F401
  gin.clear_config()
  gin.parse_config("\n".join([
      'dataset.name = "mnist"', 'options.architecture = "infogan_arch"', "options.batch_size = 16",
      "options.gan_class = @ModularGAN", "options.lamba = 1", "options.z_dim = 64", "options.disc_iters = 1",
      "D.spectral_norm = True", "loss.fn = @non_saturating", "penalty.fn = @no_penalty", "ModularGAN.g_lr = 0.0002",
      "ModularGAN.g_optimizer_fn = @tf.train.AdamOptimizer", "tf.train.AdamOptimizer.beta1 = 0.5",
      "options.training_steps = 3", "ModularGAN.math_mode = 1"]))
  md = str(tmp_path / "run")
  try:
    out = runner_lib.run_with_schedule("eval_after_train", model_dir=md, num_cycles=3, use_graph=True,
                                       input_pipeline=True, eval_kwargs=dict(num_samples=64, num_averaging_runs=1))
  finally:
    from compare_gan_b200 import kernels as K
    K.set_math_mode(0)
    gin.clear_config()
  assert out["gan"].global_step == 3
  rows = list(csv.DictReader(open(os.path.join(md, "scores.csv"))))
  assert len(rows) == 1 and rows[0]["step"] == "3"
  fid, inception = float(rows[0]["fid_score_mean"]), float(rows[0]["inception_score_mean"])
  assert np.isfinite(fid) and fid > 0 and np.isfinite(inception) and inception >= 1.0
