"""The DRAGAN and L2 discriminator penalties (reference penalty_lib.py:33-57, 85-103).

* the perturbation entry cgan_dragan_perturb against a float64 restatement: std, the stream's bits, y bit for bit, a rerun,
  graph replay, and a captured launch that follows the device step counter;
* the L2 entries over the discriminator kernel tables of resnet_cifar, resnet5 at 128x128 and BigGAN-128 at full width:
  the forward within one fp32 ulp of float64, the gradient slots bit-exact, everything else untouched;
* the oracle's restatement (tests/penalty_oracle.py): DRAGAN against central differences, L2 against its closed form;
* networks: engine vs the oracle and its float64 twin under both penalties, one math_mode 1 case, graph replay == eager,
  the kernel selection, the errors, the gin bindings, and two gloo ranks above the emulator.

The GPU bodies also run above the emulated C-ABI (tests/abi_emulator.py), with the new entries restated below."""
import contextlib
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from tests import penalty_oracle as po
from tests.abi_emulator import EmulatedLib, emulated_library, f32, i32
from tests.gpu_util import make_inputs

HERE = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------------ emulated entries

def _i64(ptr, n):
  return np.ctypeslib.as_array((ctypes.c_int64 * int(n)).from_address(int(ptr)))


def _emulated_perturb(self, y, x, n, seed, step_dev, std_out):
  xs = f32(x, n).copy()
  u = po.uniform(seed, int(i32(step_dev, 1)[0]) * n, n)
  std = po.batch_std(xs)
  f32(y, n)[:] = po.perturb(xs, u, std)
  f32(std_out, 1)[0] = std


def _segments(segs, nseg):
  t = _i64(segs, 2 * nseg).reshape(nseg, 2)
  return [(int(o), int(l)) for o, l in t]


def _emulated_l2(self, out, p, segs, nseg):
  f32(out, 1)[0] = _l2_f64(p, _segments(segs, nseg))


def _emulated_l2_bwd(self, g, p, segs, nseg, scale_dev, mul):
  c = np.float32(f32(scale_dev, 1)[0]) * np.float32(mul)
  for o, l in _segments(segs, nseg):
    dst = f32(g + 4 * o, l)
    dst[:] = dst + c * f32(p + 4 * o, l)


def _patch(setattr_fn):
  setattr_fn(EmulatedLib, "cgan_dragan_perturb", _emulated_perturb, raising=False)
  setattr_fn(EmulatedLib, "cgan_l2_penalty", _emulated_l2, raising=False)
  setattr_fn(EmulatedLib, "cgan_l2_penalty_bwd", _emulated_l2_bwd, raising=False)


@pytest.fixture(autouse=True)
def _oracle_penalties():
  with po.penalties():
    yield


@pytest.fixture
def emulated(monkeypatch):
  _patch(monkeypatch.setattr)
  with emulated_library() as lib:
    yield lib


def _l2_f64(p, segs):
  """mean over segments of sum(w^2) / 2 in float64 (p an address)."""
  return float(np.mean([0.5 * np.sum(f32(p + 4 * o, l).astype(np.float64) ** 2) for o, l in segs]))


def _step(K, value):
  return torch.tensor([value], dtype=torch.int32, device=K._RT["device"])


# ------------------------------------------------------------------------------------------ the perturbation entry

# (shape, step, near the clip edges)
PERTURB_CASES = [((4, 32, 32, 3), 3, False), ((2, 64, 64, 3), 11, False), ((64, 128, 128, 3), 7, False),
                 ((1, 5, 5, 3), 0, False), ((3, 7, 3, 5), 2, False), ((2, 16, 16, 3), 5, True)]
EMU_PERTURB = [c for c in PERTURB_CASES if np.prod(c[0]) <= 6144]


def _perturb_check(K, shape, step, edges, seed=1234):
  rng = np.random.RandomState(int(np.prod(shape)) % 1000 + step)
  x = rng.rand(*shape).astype(np.float32)
  if edges:     # most of the batch within reach of 0 and 1: the clip decides many elements
    x = np.where(rng.rand(*shape) < 0.5, 0.02 * x, 1 - 0.02 * x).astype(np.float32)
  n = x.size
  xd, y, std, counter = K.from_numpy(x), K.empty(*shape), K.empty(1), _step(K, step)
  K._call("dragan_perturb", y.ptr, xd.ptr, n, seed, counter.data_ptr(), std.ptr)
  got_y, got_std = y.cpu().copy(), std.cpu()[0]
  u = po.uniform(seed, step * n, n)
  dev_u = K.empty(n)
  K._call("random_uniform", dev_u.ptr, n, seed, step * n)
  np.testing.assert_array_equal(dev_u.cpu(), u)                      # the stream the restatement uses is the library's
  assert got_std == po.batch_std(x), (got_std, shape)
  np.testing.assert_array_equal(got_y, po.perturb(x, u, got_std).reshape(shape))
  if edges:
    assert (got_y == 0).any() and (got_y == 1).any()
  return got_y, got_std


@pytest.mark.parametrize("shape,step,edges", EMU_PERTURB)
def test_perturb_entry_on_the_emulator(emulated, shape, step, edges):
  from compare_gan_b200 import kernels as K
  _perturb_check(K, shape, step, edges)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,step,edges", PERTURB_CASES)
def test_perturb_entry_matches_float64_and_reruns_bit_identical(shape, step, edges):
  from compare_gan_b200 import kernels as K
  K.lib()
  y1, s1 = _perturb_check(K, shape, step, edges)
  y2, s2 = _perturb_check(K, shape, step, edges)
  np.testing.assert_array_equal(y1, y2)
  assert s1 == s2


@pytest.mark.gpu
def test_perturb_graph_replay_follows_the_device_counter():
  """One captured launch equals eager, and replays after the counter advanced draw the stream at the new offsets."""
  from compare_gan_b200 import kernels as K
  K.lib()
  shape, seed = (8, 32, 32, 3), 99
  n = int(np.prod(shape))
  x_np = np.random.RandomState(4).rand(*shape).astype(np.float32)
  x, y, std, step = K.from_numpy(x_np), K.empty(*shape), K.empty(1), _step(K, 5)
  K._call("dragan_perturb", y.ptr, x.ptr, n, seed, step.data_ptr(), std.ptr)
  torch.cuda.synchronize()
  eager = y.cpu().copy()
  graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream()
  with torch.cuda.stream(stream):
    K.sync_stream()
    with torch.cuda.graph(graph, stream=stream):
      K.sync_stream()
      K._call("dragan_perturb", y.ptr, x.ptr, n, seed, step.data_ptr(), std.ptr)
  torch.cuda.current_stream().wait_stream(stream)
  K.sync_stream()
  y.t.fill_(float("nan"))
  graph.replay()
  torch.cuda.synchronize()
  np.testing.assert_array_equal(y.cpu(), eager)
  sd = std.cpu()[0]
  for s in (6, 7):
    step.fill_(s)
    graph.replay()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(y.cpu(), po.perturb(x_np, po.uniform(seed, s * n, n), sd).reshape(shape))
  assert not np.array_equal(y.cpu(), eager)


# ------------------------------------------------------------------------------------------ the L2 entries

def _engine(arch, shape, batch, penalty="l2_penalty", lamba=0.1, loss="hinge", bindings=(), num_classes=0,
            conditional=False, disc_iters=1, d_lr=None, z_dim=128):
  """The engine alone (no oracle), built for `batch`."""
  from compare_gan_b200 import datasets, gin_lite as gin
  from compare_gan_b200.gans import modular_gan
  gin.clear_config()
  gin.parse_config("\n".join([
      "G.batch_norm_fn = @batch_norm", "standardize_batch.decay = 0.9", "standardize_batch.epsilon = 1e-5",
      "loss.fn = @%s" % loss, "penalty.fn = @%s" % penalty, "ModularGAN.g_lr = 0.0001",
      "ModularGAN.g_optimizer_fn = @tf.train.AdamOptimizer", "tf.train.AdamOptimizer.beta1 = 0.5",
      "tf.train.AdamOptimizer.beta2 = 0.9", "ModularGAN.conditional = %s" % conditional] + list(bindings) +
      (["ModularGAN.d_lr = %r" % d_lr] if d_lr is not None else [])))
  ds = datasets.ImageDatasetV2("synthetic", shape[0], shape[2], num_classes or None, 100)
  params = {"architecture": arch, "z_dim": z_dim, "lambda": lamba, "disc_iters": disc_iters, "seed": 0}
  return modular_gan.ModularGAN(dataset=ds, parameters=params, model_dir="/tmp/cgan_test").build(batch)


_BIGGAN = ["resnet_biggan.Discriminator.project_y = True", "G.batch_norm_fn = @conditional_batch_norm",
           "D.spectral_norm = True", "resnet_biggan.Discriminator.blocks_with_attention = 'B1'"]
L2_TABLES = {"resnet_cifar": dict(arch="resnet_cifar_arch", shape=(32, 32, 3)),
             "resnet5_128": dict(arch="resnet5_arch", shape=(128, 128, 3)),
             # BigGAN-128 at full width (ch = 96): SN, attention, projection over 1000 classes, about 88 M D parameters
             "biggan128": dict(arch="resnet_biggan_arch", shape=(128, 128, 3), z_dim=120, num_classes=1000, conditional=True,
                               bindings=_BIGGAN + ["resnet_biggan.Discriminator.ch = 96", "resnet_biggan.Generator.ch = 96"])}


def _l2_check(K, eng, seed=0):
  segs = eng.d_kernels
  flat = eng.flat_d
  rng = np.random.RandomState(seed)
  total = flat["total"]
  flat["param"].t.copy_(torch.from_numpy((0.05 * rng.standard_normal(total)).astype(np.float32)))
  prior = (rng.standard_normal(total)).astype(np.float32)
  flat["grad"].t.copy_(torch.from_numpy(prior))
  out = K.empty(1)
  K._call("l2_penalty", out.ptr, flat["param"].ptr, segs.table.data_ptr(), segs.n)
  got = out.cpu()[0]
  pairs = [flat["views"][k] for k in segs.kernels]
  p = flat["param"].cpu()
  ref = float(np.mean([0.5 * np.sum(p[o:o + l].astype(np.float64) ** 2) for o, l in pairs]))
  assert abs(float(got) - ref) <= np.spacing(np.float32(ref)), (got, ref)
  scale = K.from_numpy(np.array([0.37], np.float32))
  mul = np.float32(1.0 / segs.n)
  K._call("l2_penalty_bwd", flat["grad"].ptr, flat["param"].ptr, segs.table.data_ptr(), segs.n, scale.ptr, float(mul))
  g = flat["grad"].cpu()
  want = prior.copy()
  c = np.float32(0.37) * mul
  for o, l in pairs:
    want[o:o + l] = prior[o:o + l] + c * p[o:o + l]
  np.testing.assert_array_equal(g.view(np.uint32), want.view(np.uint32))     # kernel slots exact, the rest untouched
  return got, g


@pytest.mark.gpu
@pytest.mark.parametrize("table", sorted(L2_TABLES))
def test_l2_entries_match_float64_and_rerun_bit_identical(table):
  from compare_gan_b200 import kernels as K
  K.lib()
  eng = _engine(batch=2, **L2_TABLES[table])
  assert eng.d_kernels.n == len([k for k in eng.flat_d["views"] if k.endswith("/kernel")])
  a = _l2_check(K, eng)
  b = _l2_check(K, eng)
  assert a[0] == b[0]
  np.testing.assert_array_equal(a[1], b[1])
  if table == "biggan128":
    assert sum(eng.flat_d["views"][k][1] for k in eng.d_kernels.kernels) > 80e6


def test_l2_entries_on_the_emulator(emulated):
  from compare_gan_b200 import kernels as K
  _l2_check(K, _engine(batch=2, **L2_TABLES["resnet_cifar"]))


def test_l2_kernel_set_is_the_reference_selection(emulated):
  """Every `/kernel` of resnet_cifar's discriminator (tests/golden/resnet_cifar_variables.json, d_default) and nothing
  else: no bias, gamma / beta, u_var."""
  golden = json.load(open(os.path.join(HERE, "golden", "resnet_cifar_variables.json")))["d_default"]
  eng = _engine("resnet_cifar_arch", (32, 32, 3), 2)
  assert list(eng.d_kernels.kernels) == [k for k, _ in golden if k.endswith("/kernel")]
  assert _engine("resnet_cifar_arch", (32, 32, 3), 2, penalty="wgangp_penalty").d_kernels is None


# ------------------------------------------------------------------------------------------ the oracle's restatement

def _oracle64(arch="resnet5_arch", shape=(16, 16, 3)):
  from oracle import nets
  cfg = nets.Cfg(architecture=arch, image_shape=shape, g_bn=None)
  store = nets.VarStore(1)
  with torch.no_grad():
    nets.discriminator(store, cfg, torch.rand(2, *shape), None, True)
  for k in list(store.vars):
    v = store.vars[k].detach().double() * 5.0
    v.requires_grad_(k in store.trainable)
    store.vars[k] = v
    if k in store.trainable:
      store.trainable[k] = v
  store.dtype = torch.float64
  return cfg, store


def test_oracle_dragan_matches_central_differences():
  torch.manual_seed(0)
  cfg, store = _oracle64()
  x = torch.rand(2, 16, 16, 3, dtype=torch.float64)
  u = torch.rand(2, 16, 16, 3, dtype=torch.float64)
  w = store.vars["discriminator/B1/same_conv1/kernel"]
  gw = torch.autograd.grad(po.dragan_penalty(store, cfg, x, None, True, u), w)[0]
  for idx in ((1, 1, 3, 5), (0, 2, 1, 7)):
    eps = 1e-5
    with torch.no_grad():
      w[idx] += eps
    hi = float(po.dragan_penalty(store, cfg, x, None, True, u).detach())
    with torch.no_grad():
      w[idx] -= 2 * eps
    lo = float(po.dragan_penalty(store, cfg, x, None, True, u).detach())
    with torch.no_grad():
      w[idx] += eps
    fd = (hi - lo) / (2 * eps)
    assert abs(fd - float(gw[idx])) <= 1e-6 * max(1.0, abs(fd)), (idx, fd, float(gw[idx]))


def test_oracle_l2_is_the_closed_form():
  cfg, store = _oracle64()
  names = po.kernel_names(store)
  assert names and all(k.endswith("/kernel") for k in names)
  want = np.mean([0.5 * float((store.vars[k].detach() ** 2).sum()) for k in names])
  p = po.l2_penalty(store)
  assert abs(float(p) - want) <= 1e-12 * want
  grads = torch.autograd.grad(p, [store.vars[k] for k in names])
  for k, g in zip(names, grads):
    torch.testing.assert_close(g, store.vars[k].detach() / len(names), rtol=1e-14, atol=0)


# ------------------------------------------------------------------------------------------ networks

_DRAGAN = dict(loss="wasserstein", penalty="dragan_penalty", lamba=10.0, g_lr=1e-4, beta1=0.5, beta2=0.9)
_L2 = dict(loss="hinge", penalty="l2_penalty", lamba=0.1, g_lr=1e-4, beta1=0.5, beta2=0.9)


def _feed_draws(orc):
  """orc.cycle() fed DRAGAN's draws as the engine makes them: seed DRAGAN_SEED (replica 0), offset = the D step counter
  before each update times numel(x)."""
  from compare_gan_b200.gans import penalty_lib
  base = orc.cycle

  def cycle(images, z, labels=None, sampled_labels=None, alphas=None):
    n = images[0].size
    draws = [po.uniform(penalty_lib.DRAGAN_SEED, (orc.global_step_disc + i) * n, n).reshape(images[i].shape)
             for i in range(orc.disc_iters)]
    return base(images, z, labels, sampled_labels, draws + [None])
  orc.cycle = cycle


@contextlib.contextmanager
def _dragan_draws(*modules):
  """The make_pair of each test module returns oracles fed the engine's DRAGAN draws."""
  saved = [(m, m.make_pair) for m in modules]

  def wrap(fn):
    def make_pair(*a, **kw):
      out = fn(*a, **kw)
      for o in out[1:]:
        _feed_draws(o)
      return out
    return make_pair
  for m, fn in saved:
    m.make_pair = wrap(fn)
  try:
    yield
  finally:
    for m, fn in saved:
      m.make_pair = fn


@contextlib.contextmanager
def _d_batch_norm():
  """The oracle's discriminators with batch norm (D.batch_norm_fn = @batch_norm on the engine side)."""
  from oracle import nets as onets
  base = onets.Cfg

  class Cfg(base):
    def __init__(self, **kw):
      base.__init__(self, **kw)
      self.d_bn = "batch_norm"
  onets.Cfg = Cfg
  try:
    yield
  finally:
    onets.Cfg = base


def _run_network(arch, shape, batch, z_dim=128, num_classes=0, frozen=True, k=2, **kw):
  """_frozen_d_gradients (D weights identical on both sides: D and G gradients against float64) and two cycles of
  engine vs oracle (losses, gradients, weights after Adam, step counters), as tests/test_gan_step_gpu.py runs them."""
  from tests import test_gan_step_gpu as ts
  with _dragan_draws(ts):
    if frozen:
      ts._frozen_d_gradients(batch, shape, z_dim, k, num_classes=num_classes, tol=2e-3, arch=arch, **kw)
    eng, orc = ts.make_pair(arch, shape, batch, disc_iters=k, z_dim=z_dim, num_classes=num_classes, **kw)
    ts._cycles_both(eng, orc, batch, shape, z_dim, k, num_classes=num_classes, g_lr=kw["g_lr"], grad_tol=2e-3,
                    loss_tol=3e-3)
  return eng


def _dragan_resnet_cifar():
  _run_network("resnet_cifar_arch", (32, 32, 3), 4, **_DRAGAN)


def _dragan_resnet5():
  _run_network("resnet5_arch", (64, 64, 3), 2, **_DRAGAN)


def _dragan_sndcgan():
  _run_network("sndcgan_arch", (32, 32, 3), 4, d_sn=True, **_DRAGAN)


def _dragan_biggan():
  eb = ["resnet_biggan.Discriminator.blocks_with_attention = ''", "resnet_biggan.Generator.blocks_with_attention = ''"]
  _run_network("resnet_biggan_arch", (32, 32, 3), 4, z_dim=120, num_classes=10, ch=8, g_bn="conditional_batch_norm",
               g_sn=True, d_sn=True, sn_singular="auto", conditional=True, use_moving_averages=False, project_y=True,
               extra_bindings=eb, **_DRAGAN)


def _dragan_layer_norm():
  from tests import layer_norm_oracle as lno
  with lno.discriminator_layer_norm():
    _run_network("resnet_cifar_arch", (32, 32, 3), 4, extra_bindings=[lno.BINDING], **_DRAGAN)


def _dragan_tf32():
  import tests.test_tf32_parity_gpu as tf32_tests
  case = dict(tf32_tests.ARCHS["resnet5_wgangp"])
  case["gp"] = False
  case["pair"] = dict(case["pair"], penalty="dragan_penalty")
  tf32_tests.ARCHS["resnet5_dragan"] = case
  try:
    with _dragan_draws(tf32_tests):
      tf32_tests.test_tf32_network_parity("resnet5_dragan")
  finally:
    del tf32_tests.ARCHS["resnet5_dragan"]


def _l2_resnet_cifar_bn():
  with _d_batch_norm():
    _run_network("resnet_cifar_arch", (32, 32, 3), 4, k=1, extra_bindings=["D.batch_norm_fn = @batch_norm"], **_L2)


def _l2_biggan_attention():
  eb = ["resnet_biggan.Generator.blocks_with_attention = 'B2'", "resnet_biggan.Discriminator.blocks_with_attention = 'B1'"]
  _run_network("resnet_biggan_arch", (32, 32, 3), 4, z_dim=120, num_classes=10, ch=8, g_bn="conditional_batch_norm",
               g_sn=True, d_sn=True, sn_singular="auto", conditional=True, use_moving_averages=False, project_y=True,
               k=1, extra_bindings=eb, **_L2)


NETWORK_CASES = {"dragan_resnet_cifar": _dragan_resnet_cifar, "dragan_resnet5": _dragan_resnet5,
                 "dragan_sndcgan": _dragan_sndcgan, "dragan_biggan": _dragan_biggan,
                 "dragan_layer_norm": _dragan_layer_norm, "dragan_tf32": _dragan_tf32,
                 "l2_resnet_cifar_bn": _l2_resnet_cifar_bn, "l2_biggan_attention": _l2_biggan_attention}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(NETWORK_CASES))
def test_networks_match_the_oracle(case):
  NETWORK_CASES[case]()


@pytest.mark.parametrize("case", ["dragan_resnet_cifar", "dragan_sndcgan", "l2_resnet_cifar_bn"])
def test_networks_on_the_emulator(emulated, case):
  NETWORK_CASES[case]()
  assert emulated.launches > 0


def _ssgan_pair(**kw):
  """SSGAN engine and oracle with the rotation head, under `kw`'s loss and penalty."""
  from compare_gan_b200 import gin_lite as gin, datasets
  from compare_gan_b200.gans import modular_gan, ssgan  # noqa: F401
  from oracle import gan as ogan, nets as onets
  gin.clear_config()
  gin.parse_config("\n".join([
      "G.batch_norm_fn = @batch_norm", "standardize_batch.decay = 0.9", "standardize_batch.epsilon = 1e-5",
      "loss.fn = @%s" % kw["loss"], "penalty.fn = @%s" % kw["penalty"], "ModularGAN.g_lr = %r" % kw["g_lr"],
      "ModularGAN.g_optimizer_fn = @tf.train.AdamOptimizer", "tf.train.AdamOptimizer.beta1 = %r" % kw["beta1"],
      "tf.train.AdamOptimizer.beta2 = %r" % kw["beta2"], "SSGAN.rotated_batch_size = 8"]))
  ds = datasets.ImageDatasetV2("synthetic", 32, 3, None, 100)
  params = {"architecture": "resnet_cifar_arch", "z_dim": 128, "lambda": kw["lamba"], "disc_iters": 1, "seed": 0}
  eng = ssgan.SSGAN(dataset=ds, parameters=params, model_dir="/tmp/cgan_test").build(4)
  cfg = onets.Cfg(architecture="resnet_cifar_arch", image_shape=(32, 32, 3), g_bn="batch_norm", bn_decay=0.9,
                  bn_eps=1e-5)
  orc = ogan.SsganOracle(cfg, 8, loss=kw["loss"], penalty=kw["penalty"], lamba=kw["lamba"], g_lr=kw["g_lr"],
                         beta1=kw["beta1"], beta2=kw["beta2"]).build(4)
  orc.store.load_numpy(eng.state_numpy())
  return eng, orc


def _l2_ssgan():
  from tests.gpu_util import compare_grads
  eng, orc = _ssgan_pair(**_L2)
  assert "discriminator_rotation/score_classify/kernel" in eng.d_kernels.kernels
  assert "discriminator_rotation/score_classify/kernel" in po.kernel_names(orc.store)
  rng = np.random.RandomState(3)
  for c in range(2):
    inputs = make_inputs(rng, 1, 4, (32, 32, 3), 128)
    eng.set_inputs(*inputs)
    eng.run_cycle()
    dl, gl = eng.read_losses()
    odl, ogl = orc.cycle(*inputs)
    assert abs(dl[0] - odl[0]) <= 3e-3 * max(1.0, abs(odl[0])) and abs(gl - ogl) <= 3e-3 * max(1.0, abs(ogl))
    if c == 0:
      compare_grads(eng, orc, 2e-3, g_tol=5e-2)
  assert eng.global_step == 2 and eng.global_step_disc == 2
  # weights after Adam, in units of the step size as compare_states measures them (it keys its bounds by network name,
  # which the rotation head's scope is not)
  state = eng.state_numpy()
  grads = dict(orc.last_d_grads, **orc.last_g_grads)
  gmax = max(float(g.norm()) for g in grads.values())
  for k in orc.store.trainable:
    if float(grads[k].norm()) < 1e-4 * gmax:
      continue
    rms = float(np.sqrt(np.mean((state[k].astype(np.float64) - orc.store.vars[k].detach().numpy()) ** 2)))
    assert rms <= 0.35 * 1e-4 * 2, (k, rms)


@pytest.mark.gpu
def test_l2_ssgan_penalises_the_rotation_head():
  _l2_ssgan()


def test_l2_ssgan_on_the_emulator(emulated):
  _l2_ssgan()


# ------------------------------------------------------------------------------------------ replay and streams

def _replay_equals_eager(penalty_kw, cycles=2):
  """Eager cycles, then the captured graph from the same start: bit-identical losses and state.  Under DRAGAN each replay
  draws at the counter's new value: the replayed losses also match the oracle fed the regenerated draws."""
  from tests import test_gan_step_gpu as ts
  with _dragan_draws(ts):
    eng, orc = ts.make_pair("resnet_cifar_arch", (32, 32, 3), 4, disc_iters=2, **penalty_kw)
  rng = np.random.RandomState(9)
  batches = [make_inputs(rng, 2, 4, (32, 32, 3), 128) for _ in range(cycles)]
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
    odl, ogl = orc.cycle(*b)
    assert all(abs(a - o) <= 3e-3 * max(1.0, abs(o)) for a, o in zip(eager[i][0], odl)), (eager[i], odl)
  for k, v in eng.state_numpy().items():
    np.testing.assert_array_equal(v, state_eager[k], err_msg=k)
  assert eng.global_step_disc == 2 * cycles
  return eager


@pytest.mark.gpu
def test_dragan_graph_replay_equals_eager_and_draws_fresh_noise():
  eager = _replay_equals_eager(_DRAGAN)
  assert eager[0] != eager[1]


@pytest.mark.gpu
def test_l2_graph_replay_equals_eager():
  _replay_equals_eager(_L2)


def test_dragan_noise_follows_the_step_counter(emulated):
  """The same real batch at D steps 0 and 1 is perturbed with the stream at offsets 0 and numel(x); restoring the counter
  repeats the draw."""
  from compare_gan_b200 import kernels as K
  from compare_gan_b200.gans import penalty_lib
  x = np.random.RandomState(0).rand(2, 8, 8, 3).astype(np.float32)
  n = x.size
  step = _step(K, 0)
  outs = []
  for s in (0, 1, 0):
    step.fill_(s)
    y, std = K.dragan_perturb(K.from_numpy(x), penalty_lib.DRAGAN_SEED, step)
    outs.append(y.cpu().copy())
    np.testing.assert_array_equal(outs[-1], po.perturb(x, po.uniform(penalty_lib.DRAGAN_SEED, s * n, n),
                                                       std.cpu()[0]).reshape(x.shape))
  assert not np.array_equal(outs[0], outs[1])
  np.testing.assert_array_equal(outs[0], outs[2])


# ------------------------------------------------------------------------------------------ selection and errors

@pytest.mark.parametrize("where", ["batch_norm", "attention"])
def test_dragan_raises_where_wgangp_raises(emulated, where):
  """Batch norm or attention in the differentiated discriminator: the same NotImplementedError as WGAN-GP."""
  from tests.gpu_util import make_pair
  if where == "attention":
    kw = dict(ch=8, z_dim=120, g_bn="conditional_batch_norm", conditional=True, num_classes=10,
              extra_bindings=["resnet_biggan.Discriminator.blocks_with_attention = 'B1'"])
    arch = "resnet_biggan_arch"
  else:
    kw = dict(extra_bindings=["D.batch_norm_fn = @batch_norm"])
    arch = "resnet_cifar_arch"
  errors = []
  for penalty in ("wgangp_penalty", "dragan_penalty"):
    with (_d_batch_norm() if where == "batch_norm" else contextlib.nullcontext()):
      eng, _ = make_pair(arch, (32, 32, 3), 2, loss="wasserstein", penalty=penalty, lamba=10.0, **kw)
    eng.set_inputs(*make_inputs(np.random.RandomState(0), 1, 2, (32, 32, 3), kw.get("z_dim", 128),
                                num_classes=kw.get("num_classes", 0), gp=True))
    with pytest.raises(NotImplementedError) as e:
      eng.run_cycle()
    errors.append(str(e.value))
  assert errors[0] == errors[1]
  assert ("attention" if where == "attention" else "batch norm") in errors[1], errors[1]


def test_penalties_bind_through_gin_and_need_their_engine_arguments(emulated):
  from compare_gan_b200 import kernels as K
  from compare_gan_b200.gans import penalty_lib
  for name, fn in (("dragan_penalty", penalty_lib.dragan_penalty), ("l2_penalty", penalty_lib.l2_penalty)):
    eng = _engine("resnet_cifar_arch", (32, 32, 3), 2, penalty=name)
    assert penalty_lib.bound_penalty() is fn
    assert (eng.d_kernels is not None) == (name == "l2_penalty")
    eng.set_inputs(*make_inputs(np.random.RandomState(0), 1, 2, (32, 32, 3), 128))
    eng.run_cycle()
    dl, _ = eng.read_losses()
    assert np.isfinite(dl).all() and eng.global_step_disc == 1
  x = K.from_numpy(np.zeros((2, 8, 8, 3), np.float32))
  with pytest.raises(ValueError, match="step"):
    penalty_lib.get_penalty_loss(fn=penalty_lib.dragan_penalty, discriminator=None, x=x, x_fake=x, y=None,
                                 is_training=True)
  with pytest.raises(ValueError, match="kernel"):
    penalty_lib.get_penalty_loss(fn=penalty_lib.l2_penalty, discriminator=None, x=x, x_fake=x, y=None, is_training=True)


# ------------------------------------------------------------------------------------------ two ranks (gloo)

def _rank_worker(rank, world, port, q):
  import sys
  import torch.distributed as dist
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  torch.set_num_threads(2)
  sys.path.insert(0, os.path.dirname(HERE))
  import pytest as _pytest
  from tests import test_penalties as tp
  from compare_gan_b200.tpu import tpu_ops
  mp = _pytest.MonkeyPatch()
  tp._patch(mp.setattr)
  per = 2
  rng = np.random.RandomState(0)
  imgs = [rng.rand(per * world, 32, 32, 3).astype(np.float32) for _ in range(2)]
  zs = [rng.uniform(-1, 1, (per * world, 128)).astype(np.float32) for _ in range(2)]
  sl = slice(rank * per, (rank + 1) * per)
  out = {}
  with emulated_library() as lib:
    # DRAGAN: this rank's shard, its std and its stream (seed + rank); record the perturbed batch the penalty sees
    from compare_gan_b200 import kernels as K
    seen = []
    real = lib.cgan_dragan_perturb

    def spy(y, x, n, seed, step_dev, std_out):
      real(y, x, n, seed, step_dev, std_out)
      seen.append((f32(x, n).copy(), f32(y, n).copy(), seed, int(i32(step_dev, 1)[0]), float(f32(std_out, 1)[0])))
    lib.cgan_dragan_perturb = spy
    eng = tp._engine("resnet_cifar_arch", (32, 32, 3), per, penalty="dragan_penalty", lamba=10.0, loss="wasserstein")
    eng.set_inputs([a[sl] for a in imgs], [a[sl] for a in zs])
    eng.run_cycle()
    out["dragan"] = seen[0]
    # L2: the exchanged D gradient, penalty term included, equals the single-rank one on the concatenated batch (the term is
    # added on every rank before the sum, and the mean keeps it)
    eng = tp._engine("resnet_cifar_arch", (32, 32, 3), per, penalty="l2_penalty", lamba=0.1)
    eng.set_inputs([a[sl] for a in imgs], [a[sl] for a in zs])
    eng.run_cycle()
    out["l2_grad"] = eng.flat_d["grad"].cpu() / world
    dist.barrier()
    if rank == 0:
      tpu_ops.force_local(True)
      ref = tp._engine("resnet_cifar_arch", (32, 32, 3), per * world, penalty="l2_penalty", lamba=0.1)
      ref.set_inputs(imgs, zs)
      ref.run_cycle()
      out["l2_ref"] = ref.flat_d["grad"].cpu()
      tpu_ops.force_local(False)
  mp.undo()
  q.put((rank, out))
  dist.barrier()
  dist.destroy_process_group()


def test_two_ranks_draw_their_own_noise_and_share_the_l2_gradient():
  import torch.multiprocessing as tmp
  from tests.test_distributed_cpu import _free_port
  from compare_gan_b200.gans import penalty_lib
  ctx = tmp.get_context("spawn")
  q = ctx.Queue()
  port = _free_port()
  procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, q)) for r in range(2)]
  for p in procs:
    p.start()
  res = dict(q.get(timeout=900) for _ in range(2))
  for p in procs:
    p.join(60)
    assert p.exitcode == 0
  rng = np.random.RandomState(0)
  imgs = rng.rand(4, 32, 32, 3).astype(np.float32)
  for r in (0, 1):
    x, y, seed, step, std = res[r]["dragan"]
    np.testing.assert_array_equal(x, imgs[2 * r:2 * r + 2].ravel())
    assert seed == penalty_lib.DRAGAN_SEED + r and step == 0
    assert std == po.batch_std(x)
    np.testing.assert_array_equal(y, po.perturb(x, po.uniform(seed, 0, x.size), std))
  assert res[0]["dragan"][4] != res[1]["dragan"][4]
  np.testing.assert_array_equal(res[0]["l2_grad"], res[1]["l2_grad"])
  g, ref = res[0]["l2_grad"].astype(np.float64), res[0]["l2_ref"].astype(np.float64)
  assert np.linalg.norm(g - ref) <= 1e-4 * np.linalg.norm(ref)
