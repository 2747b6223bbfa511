"""Layer-normalised discriminators (`D.layer_norm = True`, reference arch_ops.py:448-450, resnet_ops.py:162-173,
resnet_biggan.py:123-134) and their second order under WGAN-GP.

* the oracle's convention itself: TF's stop_gradient(mean) inside tf.nn.moments changes the penalty gradient by a
  closed-form term, and without it the oracle is the exact Hessian (central differences);
* the four C entries (moments, apply, backward, double backward) against a float64 restatement at every layer-norm shape
  of resnet5 at 128x128 and of resnet_cifar, bit-identical on a rerun and between CUDA-graph replay and eager;
* networks: engine vs the oracle and its float64 twin under WGAN-GP / hinge, one math_mode 1 case, graph == eager;
* variables: names, shapes, inits, order, a TF-checkpoint round trip; the flag is ignored where the reference ignores it.

The GPU bodies also run above the emulated C-ABI (tests/abi_emulator.py), with the layer-norm entries restated below.
The oracle side of layer norm is tests/layer_norm_oracle.py."""
import numpy as np
import pytest
import torch

from oracle import nets as onets
from tests import layer_norm_oracle as lno
from tests.abi_emulator import EmulatedLib, emulated_library, f32, rna_tf32
from tests.gpu_util import make_inputs, make_pair

EPS = 1e-12


# ------------------------------------------------------------------------------------------ emulated entries (float64)

def _ln_load(x, n, span, stats):
  xs = f32(x, n * span).reshape(n, span).astype(np.float64)
  st = f32(stats, 2 * n).reshape(n, 2).astype(np.float64)
  return xs, st[:, :1], st[:, 1:]


def _chan(p, c, span):
  return np.tile(f32(p, c).astype(np.float64), span // c)[None, :]


def _emulated_moments(self, stats, x, n, span, eps):
  xs = f32(x, n * span).reshape(n, span).astype(np.float64)
  m = xs.mean(1)
  st = f32(stats, 2 * n).reshape(n, 2)
  st[:, 0] = m
  st[:, 1] = 1.0 / np.sqrt(((xs - m[:, None]) ** 2).mean(1) + np.float32(eps))


def _emulated_apply(self, y, x, n, span, c, stats, gamma, beta, act):
  xs, m, r = _ln_load(x, n, span, stats)
  o = ((xs - m) * (r * _chan(gamma, c, span)) + _chan(beta, c, span)).astype(np.float32)
  if act & 1:
    o = np.maximum(o, 0)
  if act & 0x100:
    o = rna_tf32(o)
  f32(y, n * span)[:] = o.ravel()


def _emulated_bwd(self, dx, dgamma, dbeta, g, x, n, span, c, stats, gamma, rnd):
  xs, m, r = _ln_load(x, n, span, stats)
  gs = f32(g, n * span).reshape(n, span).astype(np.float64)
  xh = (xs - m) * r
  if dgamma:
    f32(dgamma, c)[:] = (gs * xh).reshape(-1, c).sum(0)
  if dbeta:
    f32(dbeta, c)[:] = gs.reshape(-1, c).sum(0)
  if dx:
    a = _chan(gamma, c, span) * gs
    o = (r * (a - a.mean(1, keepdims=True) - xh * (a * xh).mean(1, keepdims=True))).astype(np.float32)
    f32(dx, n * span)[:] = (rna_tf32(o) if rnd else o).ravel()


def _emulated_bwd_bwd(self, d_g, d_x, d_gamma, w, g, x, n, span, c, stats, gamma, rnd):
  xs, m, r = _ln_load(x, n, span, stats)
  gs = f32(g, n * span).reshape(n, span).astype(np.float64)
  ws = f32(w, n * span).reshape(n, span).astype(np.float64)
  gm = _chan(gamma, c, span)
  xh, a = (xs - m) * r, gm * gs
  M = lambda t: t.mean(1, keepdims=True)
  abar, mm, wbar, q = M(a), M(a * xh), M(ws), M(ws * xh)
  p = ws - wbar - xh * q
  if d_g:
    f32(d_g, n * span)[:] = (gm * r * p).astype(np.float32).ravel()
  if d_gamma:
    f32(d_gamma, c)[:] = (gs * r * p).reshape(-1, c).sum(0)
  if d_x:
    o = (-r * r * (xh * (M(ws * a) - abar * wbar - 3 * mm * q) + q * (a - abar) + mm * ws)).astype(np.float32)
    f32(d_x, n * span)[:] = (rna_tf32(o) if rnd else o).ravel()


def _patch(setattr_fn):
  setattr_fn(EmulatedLib, "cgan_layer_norm_moments", _emulated_moments, raising=False)
  setattr_fn(EmulatedLib, "cgan_layer_norm_apply", _emulated_apply, raising=False)
  setattr_fn(EmulatedLib, "cgan_layer_norm_bwd", _emulated_bwd, raising=False)
  setattr_fn(EmulatedLib, "cgan_layer_norm_bwd_bwd", _emulated_bwd_bwd, raising=False)


@pytest.fixture(autouse=True)
def _oracle_layer_norm():
  """The oracle's resnet / BigGAN discriminators with layer norm, matching the engine binding lno.BINDING."""
  with lno.discriminator_layer_norm():
    yield


@pytest.fixture
def emulated(monkeypatch):
  _patch(monkeypatch.setattr)
  from compare_gan_b200 import kernels as K
  with emulated_library() as lib:
    yield lib


# ------------------------------------------------------------------------------------------ the oracle's convention

def _ln64(x, gamma, beta, stop_gradient):
  store = onets.VarStore(dtype=torch.float64)
  y = lno.layer_norm(store, x, True, "ln", stop_gradient=stop_gradient)
  with torch.no_grad():
    store.vars["ln/gamma"].copy_(gamma)
    store.vars["ln/beta"].copy_(beta)
  return lno.layer_norm(store, x, True, "ln", stop_gradient=stop_gradient), store


def test_oracle_second_order_is_tf_graph_closed_form():
  """vjp of dx w.r.t. x: TF's graph == the exact Hessian - r^2 * mean(a*xhat) * mean(w) per sample; w.r.t. g and gamma
  both agree."""
  torch.manual_seed(1)
  n, h, w, c = 3, 5, 4, 6
  x = (torch.randn(n, h, w, c, dtype=torch.float64) * 2 + 1).requires_grad_(True)
  gamma = 1 + 0.3 * torch.randn(c, dtype=torch.float64)
  beta = 0.1 * torch.randn(c, dtype=torch.float64)
  g = torch.randn(n, h, w, c, dtype=torch.float64, requires_grad=True)
  wv = torch.randn(n, h, w, c, dtype=torch.float64)
  out = {}
  for sg in (True, False):
    y, store = _ln64(x, gamma, beta, sg)
    gm = store.vars["ln/gamma"]
    dx, = torch.autograd.grad(y, x, g, create_graph=True)
    out[sg] = torch.autograd.grad(dx, (x, gm, g), wv)
  ax = (1, 2, 3)
  m = x.mean(ax, keepdim=True)
  r = torch.rsqrt(((x - m) ** 2).mean(ax, keepdim=True) + EPS)
  a, xh = gamma * g, (x - m) * r
  closed = -(r ** 2) * (a * xh).mean(ax, keepdim=True) * wv.mean(ax, keepdim=True)
  scale = float(out[False][0].abs().max())
  assert float((out[True][0] - out[False][0] - closed).abs().max()) <= 1e-13 * scale
  assert float(closed.abs().max()) > 1e-3 * scale                       # the term is not negligible
  assert float((out[True][1] - out[False][1]).abs().max()) <= 1e-13 * float(out[False][1].abs().max())
  assert float((out[True][2] - out[False][2]).abs().max()) <= 1e-13 * float(out[False][2].abs().max())


def _critic_penalty(params, x, stop_gradient):
  """conv -> LN -> relu -> conv critic; mean((|d logit / d x| - 1)^2) (penalty_lib.py:59-82)."""
  store = onets.VarStore(dtype=torch.float64)
  h = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2), params["w1"], padding=1).permute(0, 2, 3, 1)
  lno.layer_norm(store, h, True, "ln")
  store.vars["ln/gamma"] = params["gamma"]
  store.vars["ln/beta"] = params["beta"]
  h = torch.relu(lno.layer_norm(store, h, True, "ln", stop_gradient=stop_gradient))
  h = torch.nn.functional.conv2d(h.permute(0, 3, 1, 2), params["w2"], padding=1)
  logit = h.mean(dim=(1, 2, 3))
  gx, = torch.autograd.grad(logit.sum(), x, create_graph=True)
  return ((torch.sqrt(1e-4 + (gx ** 2).sum(dim=(1, 2, 3))) - 1) ** 2).mean()


def test_oracle_exact_hessian_without_stop_gradient_matches_central_differences():
  torch.manual_seed(0)
  dt = torch.float64
  params = {"w1": torch.randn(6, 3, 3, 3, dtype=dt) * 0.3, "w2": torch.randn(4, 6, 3, 3, dtype=dt) * 0.3,
            "gamma": 1 + 0.2 * torch.randn(6, dtype=dt), "beta": 0.1 * torch.randn(6, dtype=dt)}
  x = torch.rand(2, 5, 5, 3, dtype=dt, requires_grad=True)
  for p in params.values():
    p.requires_grad_(True)
  grads = {}
  for sg in (False, True):
    grads[sg] = torch.autograd.grad(_critic_penalty(params, x, sg), list(params.values()))
  step = 1e-6
  for (name, p), g_exact, g_tf in zip(params.items(), grads[False], grads[True]):
    fd = torch.zeros_like(p)
    flat = p.detach().view(-1)
    for i in range(flat.numel()):
      old = float(flat[i])
      flat[i] = old + step
      hi = float(_critic_penalty(params, x, False))
      flat[i] = old - step
      lo = float(_critic_penalty(params, x, False))
      flat[i] = old
      fd.view(-1)[i] = (hi - lo) / (2 * step)
    if name == "beta":    # reaches the penalty only through the ReLU mask: zero almost everywhere
      assert float(fd.abs().max()) < 1e-8 and float(g_exact.abs().max()) < 1e-12
      continue
    err = float((g_exact - fd).norm() / fd.norm())
    assert err < 1e-6, (name, err)
    if name == "w1":      # upstream of the LN the two conventions differ measurably
      assert float((g_tf - g_exact).norm() / g_exact.norm()) > 1e-6


# ------------------------------------------------------------------------------------------ entries

RESNET5_128 = [(128, 128, 3), (128, 128, 64), (64, 64, 64), (64, 64, 128), (32, 32, 128), (32, 32, 256), (16, 16, 256),
               (8, 8, 256), (8, 8, 512), (4, 4, 512)]
RESNET_CIFAR = [(32, 32, 3), (32, 32, 128), (16, 16, 128), (8, 8, 128)]
# (batch, h, w, c): every LN shape of both discriminators at batch 2, plus N = 1 and spans that are not multiples of 4
ENTRY_CASES = [(2,) + s for s in RESNET5_128 + RESNET_CIFAR] + [(1, 32, 32, 128), (1, 5, 5, 3), (3, 7, 3, 5)]
EMU_CASES = [(2, 8, 8, 128), (1, 5, 5, 3), (3, 7, 3, 5), (2, 16, 16, 3)]


def _entry_check(K, n, h, w, c, relu, seed=0):
  """Runs the four entries once and returns their outputs (numpy), after checking them against float64 autograd
  through the oracle's op-by-op graph."""
  rng = np.random.RandomState(seed + n * 7 + c)
  x = (rng.standard_normal((n, h, w, c)) * 1.5 + rng.standard_normal((n, 1, 1, 1)) * 3).astype(np.float32)
  gamma = (1 + 0.3 * rng.standard_normal(c)).astype(np.float32)
  beta = (0.2 * rng.standard_normal(c)).astype(np.float32)
  g = rng.standard_normal((n, h, w, c)).astype(np.float32)
  wv = rng.standard_normal((n, h, w, c)).astype(np.float32)
  span = h * w * c
  dx_, gm_, bt_, g_, w_ = (K.from_numpy(a) for a in (x, gamma, beta, g, wv))
  stats, y = K.empty(2 * n), K.empty(n, h, w, c)
  K._call("layer_norm_moments", stats.ptr, dx_.ptr, n, span, EPS)
  K._call("layer_norm_apply", y.ptr, dx_.ptr, n, span, c, stats.ptr, gm_.ptr, bt_.ptr, 1 if relu else 0)
  dx, dgamma, dbeta = K.empty(n, h, w, c), K.empty(c), K.empty(c)
  K._call("layer_norm_bwd", dx.ptr, dgamma.ptr, dbeta.ptr, g_.ptr, dx_.ptr, n, span, c, stats.ptr, gm_.ptr, 0)
  d_g, d_x, d_gamma = K.empty(n, h, w, c), K.empty(n, h, w, c), K.empty(c)
  K._call("layer_norm_bwd_bwd", d_g.ptr, d_x.ptr, d_gamma.ptr, w_.ptr, g_.ptr, dx_.ptr, n, span, c, stats.ptr, gm_.ptr, 0)
  got = {k: v.cpu().copy() for k, v in dict(stats=stats, y=y, dx=dx, dgamma=dgamma, dbeta=dbeta, d_g=d_g, d_x=d_x,
                                             d_gamma=d_gamma).items()}

  tx = torch.from_numpy(x).double().requires_grad_(True)
  tg = torch.from_numpy(g).double().requires_grad_(True)
  ty, store = _ln64(tx, torch.from_numpy(gamma).double(), torch.from_numpy(beta).double(), True)
  tgm, tbt = store.vars["ln/gamma"], store.vars["ln/beta"]
  rdx, rdgamma, rdbeta = torch.autograd.grad(ty, (tx, tgm, tbt), tg, create_graph=True)
  rd_x, rd_gamma, rd_g = torch.autograd.grad(rdx, (tx, tgm, tg), torch.from_numpy(wv).double())
  ax = (1, 2, 3)
  m = tx.detach().mean(ax)
  ref = dict(stats=torch.stack([m, torch.rsqrt(((tx.detach() - m[:, None, None, None]) ** 2).mean(ax) + EPS)], 1),
             y=torch.relu(ty) if relu else ty, dx=rdx, dgamma=rdgamma, dbeta=rdbeta, d_g=rd_g, d_x=rd_x, d_gamma=rd_gamma)
  # fp32 inputs, float64 truth: the forward and backward lose a few ulps per element, the double backward's
  # x-derivative sums several per-sample terms that partly cancel
  tols = dict(stats=2e-6, y=3e-6, dx=2e-5, dgamma=2e-5, dbeta=2e-5, d_g=2e-5, d_x=2e-4, d_gamma=2e-5)
  for k, r in ref.items():
    r = r.detach().numpy().reshape(got[k].shape)
    a = got[k].astype(np.float64)
    assert np.isfinite(a).all(), k
    err = np.linalg.norm(a - r) / max(np.linalg.norm(r), 1e-30)
    assert err <= tols[k], "%s at %s: rel-L2 %.2e > %.1e" % (k, (n, h, w, c), err, tols[k])
  return got


@pytest.mark.parametrize("n,h,w,c", EMU_CASES)
def test_entries_on_the_emulator(emulated, n, h, w, c):
  from compare_gan_b200 import kernels as K
  _entry_check(K, n, h, w, c, relu=(c % 2 == 0))


def test_taped_layer_norm_second_order_on_the_emulator(emulated):
  """K.layer_norm through the tape with create_graph (the WGAN-GP path) == torch autograd through the oracle graph."""
  from compare_gan_b200 import kernels as K, tape
  rng = np.random.RandomState(3)
  n, h, w, c = 2, 4, 4, 8
  x = rng.standard_normal((n, h, w, c)).astype(np.float32)
  gamma = (1 + 0.3 * rng.standard_normal(c)).astype(np.float32)
  beta = (0.2 * rng.standard_normal(c)).astype(np.float32)
  k = rng.standard_normal((n, h, w, c)).astype(np.float32)
  xe, ge, be = K.from_numpy(x, True), K.from_numpy(gamma, True), K.from_numpy(beta, True)
  with tape.record(True):
    y = K.layer_norm(xe, ge, be, relu_after=True)
    (gx,) = tape.backward([(y, K.from_numpy(k))], [xe], K.add_grad, create_graph=True)
    pen = K.gp_penalty(gx)
  dxe, dge, dbe = tape.backward([(pen, K.fill_(K.empty(1), 1.0))], [xe, ge, be], K.add_grad)
  tx = torch.from_numpy(x).double().requires_grad_(True)
  ty, store = _ln64(tx, torch.from_numpy(gamma).double(), torch.from_numpy(beta).double(), True)
  tgx, = torch.autograd.grad(torch.relu(ty), tx, torch.from_numpy(k).double(), create_graph=True)
  tpen = ((torch.sqrt(1e-4 + (tgx ** 2).sum(dim=(1, 2, 3))) - 1) ** 2).mean()
  ref = torch.autograd.grad(tpen, (tx, store.vars["ln/gamma"], store.vars["ln/beta"]), allow_unused=True)
  np.testing.assert_allclose(float(pen.cpu()[0]), float(tpen), rtol=1e-5)
  for got, r, name in ((dxe, ref[0], "x"), (dge, ref[1], "gamma")):
    r = r.numpy()
    assert np.linalg.norm(got.cpu() - r) <= 1e-4 * np.linalg.norm(r), name
  assert dbe is None or np.abs(dbe.cpu()).max() <= 1e-5 * np.abs(ref[0].numpy()).max()    # beta does not reach the penalty


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w,c", ENTRY_CASES)
def test_entries_match_float64_and_rerun_bit_identical(n, h, w, c):
  from compare_gan_b200 import kernels as K
  K.lib()
  first = _entry_check(K, n, h, w, c, relu=(c % 2 == 0))
  again = _entry_check(K, n, h, w, c, relu=(c % 2 == 0))
  for k in first:
    np.testing.assert_array_equal(first[k], again[k], err_msg=k)


@pytest.mark.gpu
def test_entries_graph_replay_equals_eager():
  from compare_gan_b200 import kernels as K
  K.lib()
  n, h, w, c = 4, 32, 32, 128
  span = h * w * c
  rng = np.random.RandomState(5)
  x, g, wv = (K.from_numpy(rng.standard_normal((n, h, w, c)).astype(np.float32)) for _ in range(3))
  gamma = K.from_numpy((1 + 0.3 * rng.standard_normal(c)).astype(np.float32))
  beta = K.from_numpy((0.1 * rng.standard_normal(c)).astype(np.float32))
  outs = dict(stats=K.empty(2 * n), y=K.empty(n, h, w, c), dx=K.empty(n, h, w, c), dgamma=K.empty(c), dbeta=K.empty(c),
              d_g=K.empty(n, h, w, c), d_x=K.empty(n, h, w, c), d_gamma=K.empty(c))

  def run():
    o = outs
    K._call("layer_norm_moments", o["stats"].ptr, x.ptr, n, span, EPS)
    K._call("layer_norm_apply", o["y"].ptr, x.ptr, n, span, c, o["stats"].ptr, gamma.ptr, beta.ptr, 1)
    K._call("layer_norm_bwd", o["dx"].ptr, o["dgamma"].ptr, o["dbeta"].ptr, g.ptr, x.ptr, n, span, c, o["stats"].ptr,
            gamma.ptr, 0)
    K._call("layer_norm_bwd_bwd", o["d_g"].ptr, o["d_x"].ptr, o["d_gamma"].ptr, wv.ptr, g.ptr, x.ptr, n, span, c,
            o["stats"].ptr, gamma.ptr, 0)
  run()
  torch.cuda.synchronize()
  eager = {k: v.cpu().copy() for k, v in outs.items()}
  for v in outs.values():
    v.t.fill_(float("nan"))
  graph = torch.cuda.CUDAGraph()
  stream = torch.cuda.Stream()
  with torch.cuda.stream(stream):
    K.sync_stream()
    with torch.cuda.graph(graph, stream=stream):
      K.sync_stream()
      run()
  torch.cuda.current_stream().wait_stream(stream)
  K.sync_stream()
  for _ in range(2):
    for v in outs.values():
      v.t.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    for k, v in outs.items():
      np.testing.assert_array_equal(v.cpu(), eager[k], err_msg=k)


# ------------------------------------------------------------------------------------------ networks

_WGANGP = dict(loss="wasserstein", penalty="wgangp_penalty", lamba=10.0, g_lr=1e-4, beta1=0.5, beta2=0.9)
_LN = [lno.BINDING]


def _ln_resnet_cifar_wgangp():
  from tests.test_gan_step_gpu import _cycles_both, _forward_both, _frozen_d_gradients
  _frozen_d_gradients(4, (32, 32, 3), 128, 2, gp=True, tol=2e-3, arch="resnet_cifar_arch", extra_bindings=_LN, **_WGANGP)
  eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 4, disc_iters=2, extra_bindings=_LN, **_WGANGP)
  _forward_both(eng, orc, 4, 128)
  _cycles_both(eng, orc, 4, (32, 32, 3), 128, 2, gp=True, g_lr=1e-4, grad_tol=2e-3, loss_tol=3e-3)


def _ln_resnet5_wgangp():
  from tests.test_gan_step_gpu import _cycles_both, _forward_both, _frozen_d_gradients
  _frozen_d_gradients(2, (64, 64, 3), 128, 2, gp=True, tol=2e-3, arch="resnet5_arch", extra_bindings=_LN, **_WGANGP)
  eng, orc = make_pair("resnet5_arch", (64, 64, 3), 2, disc_iters=2, extra_bindings=_LN, **_WGANGP)
  _forward_both(eng, orc, 2, 128)
  _cycles_both(eng, orc, 2, (64, 64, 3), 128, 2, gp=True, g_lr=1e-4, grad_tol=2e-3, loss_tol=3e-3)


def _ln_biggan_wgangp():
  from tests.test_gan_step_gpu import _cycles_both, _forward_both, _frozen_d_gradients
  # conditional G with accumulators (BigGAN's G embeds y), attention off on both sides, no projection in D
  kw = dict(arch="resnet_biggan_arch", ch=8, g_bn="conditional_batch_norm", conditional=True,
            use_moving_averages=False, **_WGANGP)
  eb = _LN + ["resnet_biggan.Discriminator.blocks_with_attention = ''",
               "resnet_biggan.Generator.blocks_with_attention = ''"]
  _frozen_d_gradients(4, (32, 32, 3), 120, 2, num_classes=10, gp=True, tol=2e-3, extra_bindings=eb, **kw)
  kw.pop("arch")
  eng, orc = make_pair("resnet_biggan_arch", (32, 32, 3), 4, disc_iters=2, z_dim=120, num_classes=10, extra_bindings=eb,
                       **kw)
  _forward_both(eng, orc, 4, 120, num_classes=10)
  _cycles_both(eng, orc, 4, (32, 32, 3), 120, 2, num_classes=10, gp=True, g_lr=1e-4, grad_tol=2e-3, loss_tol=3e-3)


def _ln_resnet_cifar_hinge():
  from tests.test_gan_step_gpu import _cycles_both, _frozen_d_gradients
  _frozen_d_gradients(4, (32, 32, 3), 128, 1, arch="resnet_cifar_arch", loss="hinge", extra_bindings=_LN)
  eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 4, loss="hinge", disc_iters=1, extra_bindings=_LN)
  _cycles_both(eng, orc, 4, (32, 32, 3), 128, 1)


def _ln_resnet5_tf32():
  import tests.test_tf32_parity_gpu as tf32_tests
  case = dict(tf32_tests.ARCHS["resnet5_wgangp"])
  case["pair"] = dict(case["pair"], extra_bindings=_LN)
  tf32_tests.ARCHS["resnet5_wgangp_ln"] = case
  try:
    tf32_tests.test_tf32_network_parity("resnet5_wgangp_ln")
  finally:
    del tf32_tests.ARCHS["resnet5_wgangp_ln"]


def _ln_graph_replay_equals_eager():
  from compare_gan_b200 import kernels as K
  eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 4, disc_iters=2, extra_bindings=_LN, **_WGANGP)
  rng = np.random.RandomState(9)
  batches = [make_inputs(rng, 2, 4, (32, 32, 3), 128, gp=True) for _ in range(2)]
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


NETWORK_CASES = {"resnet_cifar_wgangp": _ln_resnet_cifar_wgangp, "resnet5_wgangp": _ln_resnet5_wgangp,
                 "biggan_wgangp": _ln_biggan_wgangp, "resnet_cifar_hinge": _ln_resnet_cifar_hinge,
                 "resnet5_tf32": _ln_resnet5_tf32}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(NETWORK_CASES))
def test_layer_norm_networks_match_the_oracle(case):
  NETWORK_CASES[case]()


@pytest.mark.gpu
def test_layer_norm_cycle_graph_replay_equals_eager():
  _ln_graph_replay_equals_eager()


@pytest.mark.parametrize("case", ["resnet_cifar_wgangp", "biggan_wgangp", "resnet_cifar_hinge", "resnet5_tf32"])
def test_layer_norm_networks_on_the_emulator(emulated, case):
  NETWORK_CASES[case]()
  assert emulated.launches > 0


# ------------------------------------------------------------------------------------------ variables

def test_variables_names_inits_order_and_checkpoint_round_trip(emulated, tmp_path):
  from compare_gan_b200 import tf_checkpoint as tfc
  eng, orc = make_pair("resnet5_arch", (64, 64, 3), 2, extra_bindings=_LN, **_WGANGP)    # asserts equal sets and trainable order
  names = list(eng.store.trainable)
  state = eng.state_numpy()
  for blk, cin, cout in (("B0", 3, 64), ("B1", 64, 128), ("B5", 512, 512)):
    for ln, c in (("ln1", cin), ("ln2", cout)):
      beta, gamma = "discriminator/%s/%s/beta" % (blk, ln), "discriminator/%s/%s/gamma" % (blk, ln)
      assert state[beta].shape == (c,) and state[gamma].shape == (c,)
      assert not state[beta].any() and (state[gamma] == 1).all()
      assert names.index(beta) + 1 == names.index(gamma)
  order = [k for k in names if k.startswith("discriminator/B1/")]
  assert order == ["discriminator/B1/down_conv_shortcut/kernel", "discriminator/B1/down_conv_shortcut/bias",
                   "discriminator/B1/ln1/beta", "discriminator/B1/ln1/gamma",
                   "discriminator/B1/same_conv1/kernel", "discriminator/B1/same_conv1/bias",
                   "discriminator/B1/ln2/beta", "discriminator/B1/ln2/gamma",
                   "discriminator/B1/down_conv2/kernel", "discriminator/B1/down_conv2/bias"], order
  assert not any("/ln" in k for k in names if k.startswith("generator/"))
  eng.set_inputs(*make_inputs(np.random.RandomState(0), 2, 2, (64, 64, 3), 128, gp=True))
  eng.run_cycle()
  eng.read_losses()
  want = eng.checkpoint_dict()
  assert "discriminator/B2/ln2/gamma/Adam" in want
  prefix = tfc.save_checkpoint(str(tmp_path / "model.ckpt-1"), want)
  eng.store.vars["discriminator/B2/ln2/gamma"].t.zero_()
  eng.load_checkpoint(prefix)
  got = eng.checkpoint_dict()
  for k in want:
    np.testing.assert_array_equal(got[k], want[k], err_msg=k)


@pytest.mark.parametrize("arch", ["dcgan_arch", "sndcgan_arch", "resnet_biggan_deep_arch"])
def test_flag_is_ignored_where_the_reference_ignores_it(emulated, arch):
  from compare_gan_b200 import kernels as K, tape, variables as V
  runs = []
  deep = arch == "resnet_biggan_deep_arch"
  shape = (64, 64, 3) if deep else (32, 32, 3)
  kw = dict(g_bn="conditional_batch_norm", conditional=True, num_classes=10, ch=4) if deep else {}
  for ln in (False, True):
    eng, _ = make_pair(arch, shape, 2, extra_bindings=_LN if ln else [], **kw)
    calls = []
    lib = K._RT["lib"]
    real = lib.call
    lib.call = lambda name, *args: (calls.append(name), real(name, *args))
    try:
      with V.use(eng.store), tape.no_record():
        x = K.from_numpy(np.random.RandomState(0).rand(2, *shape).astype(np.float32))
        eng.discriminator(x, y=None, is_training=True)
    finally:
      lib.call = real
    runs.append(({k: v.shape for k, v in eng.state_numpy().items()}, list(eng.store.trainable), calls))
  assert runs[0] == runs[1]
  assert not any("layer_norm" in c for c in runs[1][2])


def test_biggan_attention_under_a_gradient_penalty_still_raises(emulated):
  eng, _ = make_pair("resnet_biggan_arch", (32, 32, 3), 2, ch=8, z_dim=120, g_bn="conditional_batch_norm",
                     conditional=True, num_classes=10,
                     extra_bindings=_LN + ["resnet_biggan.Discriminator.blocks_with_attention = 'B1'"], **_WGANGP)
  eng.set_inputs(*make_inputs(np.random.RandomState(0), 1, 2, (32, 32, 3), 120, num_classes=10, gp=True))
  with pytest.raises(NotImplementedError, match="attention"):
    eng.run_cycle()
