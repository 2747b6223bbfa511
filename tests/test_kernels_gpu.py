"""Per-op parity: every C-ABI kernel family against the CPU oracle on the same seeded inputs.
Tolerances: fp32 SIMT path 2e-5 rel-L2 (reduction order only); stated per test otherwise."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import gan as ogan
from oracle import metrics as ometrics
from oracle import tf_ops as T
from tests.gpu_util import assert_close

pytestmark = pytest.mark.gpu

TOL = 2e-5


@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  return kernels


def dev(K, a, req=False):
  return K.from_numpy(np.asarray(a, np.float32), req=req)


def tape_grads(K, out, seed, wrt):
  from compare_gan_b200 import tape
  return tape.backward([(out, dev(K, seed))], wrt, K.add)


CONV_CASES = [
    # n, h, cin, cout, k, stride, upsample
    (2, 8, 3, 16, 3, 1, False),
    (2, 8, 16, 32, 3, 1, False),
    (3, 4, 8, 8, 3, 1, True),
    (2, 8, 16, 24, 4, 2, False),
    (2, 8, 16, 16, 1, 1, False),
    (3, 10, 3, 96, 1, 1, False),       # pointwise conv over image channels (BigGAN D B1 shortcut): the streaming 1x1 kernels
    (2, 7, 4, 20, 1, 1, False),
    (2, 4, 8, 8, 1, 1, True),
    (2, 9, 5, 7, 5, 2, False),
    (2, 8, 32, 3, 3, 1, False),
    (2, 16, 40, 136, 3, 1, False),
    (1, 6, 8, 200, 3, 1, False),
    # the generator shapes of resnet_cifar at batch 4
    (4, 4, 256, 256, 3, 1, True),
    (4, 16, 256, 256, 3, 1, True),
    (4, 32, 256, 256, 3, 1, False),
    (4, 32, 256, 3, 3, 1, False),
]


@pytest.mark.parametrize("n,h,cin,cout,k,stride,up", CONV_CASES)
def test_conv2d_fwd_dgrad_wgrad(K, n, h, cin, cout, k, stride, up):
  rng = np.random.RandomState(hash((n, h, cin, cout, k, stride, up)) % 2**31)
  x = rng.randn(n, h, h, cin).astype(np.float32)
  w = (rng.randn(k, k, cin, cout) * 0.1).astype(np.float32)
  b = rng.randn(cout).astype(np.float32)
  xt = torch.from_numpy(x).requires_grad_(True)
  wt = torch.from_numpy(w).requires_grad_(True)
  bt = torch.from_numpy(b).requires_grad_(True)
  ref = T.conv2d_same(T.unpool(xt) if up else xt, wt, stride) + bt
  gy = rng.randn(*ref.shape).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  xd, wd, bd = dev(K, x, True), dev(K, w, True), dev(K, b, True)
  y = K.conv2d(xd, wd, bd, stride=stride, upsample=up)
  assert_close(y.cpu(), ref.detach().numpy(), TOL, "conv fwd")
  gx, gw, gb = tape_grads(K, y, gy, [xd, wd, bd])
  assert_close(gx.cpu(), xt.grad.numpy(), TOL, "conv dgrad")
  assert_close(gw.cpu(), wt.grad.numpy(), TOL, "conv wgrad")
  assert_close(gb.cpu(), bt.grad.numpy(), TOL, "conv bias grad")


@pytest.mark.parametrize("mode,n,h,cin,cout,k,up", [
    (0, 3, 10, 3, 96, 1, False),        # pointwise stream kernel (residual fused in the kernel)
    (0, 2, 12, 3, 32, 3, False),        # 3x3 image-side kernel + post pass
    (0, 2, 8, 16, 24, 3, False),        # exact fp32 SIMT + post pass
    (1, 4, 16, 64, 64, 3, False),       # tensor-core epilogue
    (1, 4, 8, 64, 96, 3, True),         # tensor cores, sub-pixel phases
    (1, 4, 8, 64, 64, 1, True),         # 1x1 over the zero-inserted input (phase 0 + bias phases + post pass)
])
def test_conv2d_fused_epilogue(K, mode, n, h, cin, cout, k, up):
  """conv2d(..., relu, residual) == relu(conv2d(...) + residual) on every forward path, and the gradients flow to the
  residual, the input and the filter as in the unfused composition."""
  from compare_gan_b200 import tape
  rng = np.random.RandomState(cin * cout + k)
  x = rng.randn(n, h, h, cin).astype(np.float32)
  w = (rng.randn(k, k, cin, cout) * 0.1).astype(np.float32)
  b = rng.randn(cout).astype(np.float32)
  oh = 2 * h if up else h
  r = rng.randn(n, oh, oh, cout).astype(np.float32)
  gy = rng.randn(n, oh, oh, cout).astype(np.float32)
  K.set_math_mode(mode)
  try:
    outs = []
    for fused in (True, False):
      xd, wd, bd, rd = dev(K, x, True), dev(K, w, True), dev(K, b, True), dev(K, r, True)
      if fused:
        y = K.conv2d(xd, wd, bd, upsample=up, relu=True, residual=rd)
      else:
        y = K.relu(K.add(K.conv2d(xd, wd, bd, upsample=up), rd))
      grads = tape_grads(K, y, gy, [xd, wd, bd, rd])
      outs.append([y.cpu()] + [g.cpu() for g in grads])
  finally:
    K.set_math_mode(0)
  for a, c, what in zip(outs[0], outs[1], ("output", "dx", "dw", "dbias", "dresidual")):
    # math_mode 1: the fused path hands the ReLU gradient to the contractions TF32-rounded (3e-4 operand noise)
    assert_close(a, c, 1e-5 if mode == 0 else 1e-3, "fused vs composed " + what)
  xt = torch.from_numpy(x)
  ref = torch.relu(T.conv2d_same(T.unpool(xt) if up else xt, torch.from_numpy(w), 1) + torch.from_numpy(b) + torch.from_numpy(r))
  assert_close(outs[0][0], ref.numpy(), TOL if mode == 0 else 2e-3, "fused conv epilogue vs oracle")


@pytest.mark.parametrize("k,stride,h", [(4, 2, 4), (3, 1, 6), (5, 2, 5)])
def test_deconv2d(K, k, stride, h):
  rng = np.random.RandomState(k * 10 + stride)
  n, cin, cout = 2, 16, 8
  oh = h * stride
  x = rng.randn(n, h, h, cin).astype(np.float32)
  w = (rng.randn(k, k, cout, cin) * 0.1).astype(np.float32)
  b = rng.randn(cout).astype(np.float32)
  xt, wt = torch.from_numpy(x).requires_grad_(True), torch.from_numpy(w).requires_grad_(True)
  ref = T.conv2d_transpose_same(xt, wt, (oh, oh), stride) + torch.from_numpy(b)
  gy = rng.randn(*ref.shape).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  xd, wd, bd = dev(K, x, True), dev(K, w, True), dev(K, b, True)
  y = K.deconv2d(xd, wd, bd, (oh, oh), stride)
  assert_close(y.cpu(), ref.detach().numpy(), TOL, "deconv fwd")
  gx, gw, gb = tape_grads(K, y, gy, [xd, wd, bd])
  assert_close(gx.cpu(), xt.grad.numpy(), TOL, "deconv dx")
  assert_close(gw.cpu(), wt.grad.numpy(), TOL, "deconv dw")
  assert_close(gb.cpu(), gy.sum((0, 1, 2)), TOL, "deconv db")


@pytest.mark.parametrize("ta,tb", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("m,n,k", [(5, 7, 3), (64, 130, 20), (256, 4096, 128), (33, 1, 257)])
def test_matmul(K, ta, tb, m, n, k):
  rng = np.random.RandomState(m + n + k)
  a = rng.randn(*((k, m) if ta else (m, k))).astype(np.float32)
  b = rng.randn(*((n, k) if tb else (k, n))).astype(np.float32)
  at, bt = torch.from_numpy(a).requires_grad_(True), torch.from_numpy(b).requires_grad_(True)
  ref = (at.t() if ta else at) @ (bt.t() if tb else bt)
  gy = rng.randn(m, n).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  ad, bd = dev(K, a, True), dev(K, b, True)
  c = K.matmul(ad, bd, ta, tb)
  assert_close(c.cpu(), ref.detach().numpy(), TOL, "matmul")
  ga, gb = tape_grads(K, c, gy, [ad, bd])
  assert_close(ga.cpu(), at.grad.numpy(), TOL, "matmul dA")
  assert_close(gb.cpu(), bt.grad.numpy(), TOL, "matmul dB")


def test_bmm_attention_shapes(K):
  rng = np.random.RandomState(0)
  theta = rng.randn(3, 64, 6).astype(np.float32)
  phi = rng.randn(3, 16, 6).astype(np.float32)
  tt, pt = torch.from_numpy(theta).requires_grad_(True), torch.from_numpy(phi).requires_grad_(True)
  ref = torch.softmax(tt @ pt.transpose(1, 2), -1)
  gy = rng.randn(3, 64, 16).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  td, pd = dev(K, theta, True), dev(K, phi, True)
  out = K.softmax(K.bmm(td, pd, False, True))
  assert_close(out.cpu(), ref.detach().numpy(), TOL, "bmm+softmax")
  gt, gp = tape_grads(K, out, gy, [td, pd])
  assert_close(gt.cpu(), tt.grad.numpy(), 1e-4, "d theta")
  assert_close(gp.cpu(), pt.grad.numpy(), 1e-4, "d phi")


@pytest.mark.parametrize("shape,cond", [((4, 8, 8, 16), False), ((6, 4, 4, 40), True), ((16, 70), False),
                                        ((3, 16, 16, 3), False), ((4, 4, 4, 256), False),
                                        ((4, 16, 16, 256), False), ((4, 32, 32, 256), False)])
def test_bn_train(K, shape, cond):
  rng = np.random.RandomState(len(shape) + shape[-1])
  c, n = shape[-1], shape[0]
  x = (rng.randn(*shape) * 2 + 1).astype(np.float32)
  gshape = (n, c) if cond else (c,)
  gamma = (1 + 0.1 * rng.randn(*gshape)).astype(np.float32)
  beta = (0.1 * rng.randn(*gshape)).astype(np.float32)
  eps = 1e-5
  xt = torch.from_numpy(x).requires_grad_(True)
  gt, bt = torch.from_numpy(gamma).requires_grad_(True), torch.from_numpy(beta).requires_grad_(True)
  x4 = xt.reshape(-1, 1, 1, c) if len(shape) == 2 else xt
  mean, var = T.batch_moments(x4)
  yn = T.normalize(x4, mean, var, eps).reshape(shape)
  if cond:
    ref = yn * gt.reshape(n, 1, 1, c) + bt.reshape(n, 1, 1, c)
  else:
    ref = yn * gt + bt
  gy = rng.randn(*shape).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  st = K.BNState()
  st.moving_mean, st.moving_var = dev(K, np.zeros(c)), dev(K, np.ones(c))
  xd, gd, bd = dev(K, x, True), dev(K, gamma, True), dev(K, beta, True)
  y = K.bn_train(xd, gd, bd, eps, st, decay=0.9, cond=cond)
  assert_close(y.cpu(), ref.detach().numpy(), 1e-5, "bn fwd")
  assert_close(st.moving_mean.cpu(), 0.1 * mean.detach().numpy(), 1e-5, "moving mean")
  assert_close(st.moving_var.cpu(), 0.9 + 0.1 * var.detach().numpy(), 1e-5, "moving var")
  gx, gg, gb = tape_grads(K, y, gy, [xd, gd, bd])
  assert_close(gx.cpu(), xt.grad.numpy(), 5e-5, "bn dx")
  assert_close(gg.cpu(), gt.grad.numpy(), 5e-5, "bn dgamma")
  assert_close(gb.cpu(), bt.grad.numpy(), 5e-5, "bn dbeta")


def test_bn_golden_tensor(K):
  # reference architectures/arch_ops_test.py:29-61 through the CUDA kernels
  import json, os
  G = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_goldens.json")))
  x = np.array(G["bn_input"]["x"], np.float32)
  y = K.bn_train(dev(K, x), dev(K, np.ones(3)), dev(K, np.zeros(3)), 1e-3)
  np.testing.assert_allclose(y.cpu(), np.array(G["bn_expected"]["y"], np.float32), rtol=1e-5, atol=1e-5)


def test_bn_infer_accumulators(K):
  # accumulator state machine (reference arch_ops_test.py:91-132) on the device kernels
  st = K.BNState()
  st.accu_mean, st.accu_var = dev(K, np.zeros(2)), dev(K, np.zeros(2))
  st.accu_counter, st.update_accus = dev(K, np.array(1e-12)), dev(K, np.array(1.0))

  def feed(mean, var):
    m, v = np.array(mean, np.float32), np.array(var, np.float32)
    x = np.stack([m - np.sqrt(v), m + np.sqrt(v)]).reshape(2, 1, 1, 2).astype(np.float32)
    y = K.bn_infer(dev(K, x), None, None, 0.0, st, use_moving_averages=False).cpu()
    inv = (y[1, 0, 0] - y[0, 0, 0]) / (x[1, 0, 0] - x[0, 0, 0])
    return x[0, 0, 0] - y[0, 0, 0] / inv, 1.0 / inv ** 2
  m, v = feed([1., 2.], [3., 4.])
  np.testing.assert_allclose(m, [1., 2.], rtol=1e-4); np.testing.assert_allclose(v, [3., 4.], rtol=1e-4)
  m, v = feed([5., 6.], [7., 8.])
  np.testing.assert_allclose(m, [3., 4.], rtol=1e-4); np.testing.assert_allclose(v, [5., 6.], rtol=1e-4)
  K.fill_(st.update_accus, 0.0)
  m, v = feed([2., 2.], [3., 3.])
  np.testing.assert_allclose(m, [3., 4.], rtol=1e-4); np.testing.assert_allclose(v, [5., 6.], rtol=1e-4)
  np.testing.assert_allclose(st.accu_mean.cpu(), [6., 8.], rtol=1e-5)
  np.testing.assert_allclose(st.accu_var.cpu(), [10., 12.], rtol=1e-5)
  np.testing.assert_allclose(float(st.accu_counter.cpu()), 2.0, rtol=1e-6)


@pytest.mark.parametrize("shape,left", [((3, 3, 8, 16), True), ((3, 3, 16, 8), False), ((128, 4096), True),
                                        ((1024, 1), True), ((20, 64), False)])
def test_spectral_norm(K, shape, left):
  rng = np.random.RandomState(shape[-1])
  w = (rng.randn(*shape) * 0.05).astype(np.float32)
  rows, cols = int(np.prod(shape[:-1])), shape[-1]
  u0 = rng.randn(*((rows, 1) if left else (1, cols))).astype(np.float32)
  wt = torch.from_numpy(w).requires_grad_(True)
  sigma, u_new, v = T.spectral_sigma(wt.reshape(rows, cols), torch.from_numpy(u0), "left" if left else "right")
  ref = wt / sigma
  gy = rng.randn(*shape).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  wd, ud = dev(K, w, True), dev(K, u0)
  wbar = K.spectral_normalize(wd, ud, left)
  assert_close(wbar.cpu(), ref.detach().numpy(), 2e-5, "wbar")
  assert_close(ud.cpu(), u_new.numpy(), 2e-5, "u update")
  (gw,) = tape_grads(K, wbar, gy, [wd])
  assert_close(gw.cpu(), wt.grad.numpy(), 1e-4, "sn backward")


def test_pointwise_and_pools(K):
  rng = np.random.RandomState(1)
  x = rng.randn(3, 8, 8, 12).astype(np.float32)
  gy = rng.randn(3, 8, 8, 12).astype(np.float32)
  for name, fn, ref_fn in [("relu", K.relu, torch.relu), ("lrelu", lambda t: K.lrelu(t, 0.1), lambda t: T.lrelu(t, 0.1)),
                           ("sigmoid", K.sigmoid, torch.sigmoid), ("tanh01", K.tanh01, lambda t: (torch.tanh(t) + 1) / 2),
                           ("affine", lambda t: K.affine(t, 2.0, -1.0), lambda t: t * 2.0 - 1.0)]:
    xt = torch.from_numpy(x).requires_grad_(True)
    ref = ref_fn(xt)
    ref.backward(torch.from_numpy(gy))
    xd = dev(K, x, True)
    y = fn(xd)
    assert_close(y.cpu(), ref.detach().numpy(), 1e-6, name)
    (gx,) = tape_grads(K, y, gy, [xd])
    assert_close(gx.cpu(), xt.grad.numpy(), 1e-5, name + " grad")
  for name, fn, ref_fn in [("avgpool", K.avgpool2, T.avg_pool2), ("maxpool", K.maxpool2, T.max_pool2),
                           ("gmean", lambda t: K.globalpool(t, True), lambda t: t.mean((1, 2))),
                           ("gsum", lambda t: K.globalpool(t, False), lambda t: t.sum((1, 2)))]:
    xt = torch.from_numpy(x).requires_grad_(True)
    ref = ref_fn(xt)
    g2 = rng.randn(*ref.shape).astype(np.float32)
    ref.backward(torch.from_numpy(g2))
    xd = dev(K, x, True)
    y = fn(xd)
    assert_close(y.cpu(), ref.detach().numpy(), 1e-5, name)
    (gx,) = tape_grads(K, y, g2, [xd])
    assert_close(gx.cpu(), xt.grad.numpy(), 1e-5, name + " grad")


def test_concat_slice_onehot_rowdot(K):
  rng = np.random.RandomState(2)
  a, b = rng.randn(4, 6).astype(np.float32), rng.randn(4, 3).astype(np.float32)
  ad, bd = dev(K, a, True), dev(K, b, True)
  cc = K.concat_cols(ad, bd)
  assert_close(cc.cpu(), np.concatenate([a, b], 1), 0, "concat_cols")
  g = rng.randn(4, 9).astype(np.float32)
  ga, gb = tape_grads(K, cc, g, [ad, bd])
  assert_close(ga.cpu(), g[:, :6], 0, "concat grad a"); assert_close(gb.cpu(), g[:, 6:], 0, "concat grad b")
  s = K.slice_cols(ad, 2, 5)
  assert_close(s.cpu(), a[:, 2:5], 0, "slice_cols")
  (gs,) = tape_grads(K, s, g[:, :3], [ad])
  full = np.zeros_like(a); full[:, 2:5] = g[:, :3]
  assert_close(gs.cpu(), full, 0, "slice grad")
  labels = np.array([1, 0, 3, 2], np.int32)
  from compare_gan_b200.tape import DT
  oh = K.one_hot(DT(torch.from_numpy(labels).to(K._RT["device"])), 5)
  assert_close(oh.cpu(), np.eye(5, dtype=np.float32)[labels], 0, "one_hot")
  c = rng.randn(4, 6).astype(np.float32)
  cd = dev(K, c, True)
  rd = K.rowdot(ad, cd)
  assert_close(rd.cpu(), (a * c).sum(1, keepdims=True), 1e-6, "rowdot")
  gr = rng.randn(4, 1).astype(np.float32)
  g1, g2 = tape_grads(K, rd, gr, [ad, cd])
  assert_close(g1.cpu(), c * gr, 1e-6, "rowdot da"); assert_close(g2.cpu(), a * gr, 1e-6, "rowdot db")
  r0 = K.concat_rows(ad, cd)
  assert_close(r0.cpu(), np.concatenate([a, c], 0), 0, "concat_rows")
  x4 = rng.randn(3, 2, 2, 5).astype(np.float32)
  sg = dev(K, np.array(0.7, np.float32), True)
  xd = dev(K, x4, True)
  y = K.scale_by_param(xd, sg)
  assert_close(y.cpu(), x4 * 0.7, 1e-6, "scale_by_param")
  gy = rng.randn(3, 2, 2, 5).astype(np.float32)
  gx, gsig = tape_grads(K, y, gy, [xd, sg])
  assert_close(gx.cpu(), gy * 0.7, 1e-6, "scale dx")
  assert_close(gsig.cpu(), np.array((gy * x4).sum(), np.float32), 1e-5, "scale dsigma")


@pytest.mark.parametrize("kind", ["non_saturating", "hinge", "wasserstein", "least_squares"])
def test_losses(K, kind):
  rng = np.random.RandomState(3)
  b = 37
  lr_, lf_ = rng.randn(b, 1).astype(np.float32) * 2, rng.randn(b, 1).astype(np.float32) * 2
  for which in (0, 1):
    rt, ft = torch.from_numpy(lr_).requires_grad_(True), torch.from_numpy(lf_).requires_grad_(True)
    losses = ogan.get_losses(kind, torch.sigmoid(rt), torch.sigmoid(ft), rt, ft)
    target = losses[0] if which == 0 else losses[3]
    grads = torch.autograd.grad(target, [rt, ft], allow_unused=True)
    rd, fd = dev(K, lr_, True), dev(K, lf_, True)
    out = K.gan_losses(kind, rd, fd)
    for i in range(4):
      assert_close(out[i].cpu(), np.array([float(losses[i])], np.float32), 1e-5, "%s out%d" % (kind, i))
    g = tape_grads(K, out[0] if which == 0 else out[3], np.ones(1, np.float32), [rd, fd])
    for gi, ri, nm in zip(g, grads, ("real", "fake")):
      refg = np.zeros((b, 1), np.float32) if ri is None else ri.numpy()
      got = np.zeros((b, 1), np.float32) if gi is None else gi.cpu()
      assert np.abs(got - refg).max() <= 1e-6 + 1e-5 * np.abs(refg).max(), (kind, which, nm)


def test_gp_penalty(K):
  rng = np.random.RandomState(4)
  g = rng.randn(5, 4, 4, 3).astype(np.float32) * 0.3
  gt = torch.from_numpy(g).requires_grad_(True)
  slopes = torch.sqrt(0.0001 + (gt * gt).sum((1, 2, 3)))
  pen = ((slopes - 1.0) ** 2).mean()
  pen.backward()
  gd = dev(K, g, True)
  p = K.gp_penalty(gd)
  assert_close(p.cpu(), np.array([float(pen)], np.float32), 1e-5, "penalty")
  (dg,) = tape_grads(K, p, np.ones(1, np.float32), [gd])
  assert_close(dg.cpu(), gt.grad.numpy(), 1e-5, "penalty grad")


def test_adam_and_ema(K):
  rng = np.random.RandomState(5)
  n = 1000
  p0, g1, g2 = rng.randn(n).astype(np.float32), rng.randn(n).astype(np.float32), rng.randn(n).astype(np.float32)
  pt = torch.from_numpy(p0.copy())
  opt = ogan.TFAdam({"p": pt}, 2e-4, 0.5, 0.999)
  pd = dev(K, p0)
  m, v = K.zeros(n), K.zeros(n)
  ema = dev(K, p0)
  step = torch.zeros(1, dtype=torch.int32, device=K._RT["device"])
  ema_ref = p0.copy()
  for i, g in enumerate((g1, g2)):
    opt.step({"p": torch.from_numpy(g)})
    gd = dev(K, g * 2)          # held until the call returns (a temporary's storage may be recycled)
    K._call("adam_step", pd.ptr, gd.ptr, m.ptr, v.ptr, n, 2e-4, 0.5, 0.999, 1e-8, 0.5, step.data_ptr(),
            ema.ptr, 0.9, 1)
    decay = 0.9 * float(i >= 1)
    ema_ref = ema_ref - (ema_ref - pt.numpy()) * (1 - decay)
  assert int(step.item()) == 2
  assert_close(pd.cpu(), pt.numpy(), 1e-6, "adam params")
  assert_close(ema.cpu(), ema_ref, 1e-6, "ema")


def test_interpolate_colsum_bias(K):
  rng = np.random.RandomState(6)
  x, xf = rng.rand(4, 3, 3, 2).astype(np.float32), rng.rand(4, 3, 3, 2).astype(np.float32)
  al = rng.rand(4, 1, 1, 1).astype(np.float32)
  y = K.interpolate(dev(K, x), dev(K, xf), dev(K, al))
  assert_close(y.cpu(), x + al * (xf - x), 1e-6, "interpolate")
  big = rng.randn(5000, 37).astype(np.float32)
  assert_close(K.colsum(dev(K, big)).cpu(), big.sum(0), 1e-5, "colsum")
  assert_close(K.colsum(dev(K, big), groups=5).cpu(), big.reshape(5, 1000, 37).sum(1), 1e-5, "grouped colsum")


def test_cov_accumulate_and_fid(K):
  rng = np.random.RandomState(7)
  n, d = 300, 70
  acts = [rng.randn(n, d).astype(np.float32) + 0.3 * i for i in range(2)]
  s = torch.zeros(d, dtype=torch.float64, device=K._RT["device"])
  sxx = torch.zeros(d, d, dtype=torch.float64, device=K._RT["device"])
  for a in acts:
    ad = dev(K, a)              # held until the call returns
    K._call("cov_accumulate", ad.ptr, n, d, s.data_ptr(), sxx.data_ptr())
  allact = np.concatenate(acts).astype(np.float64)
  np.testing.assert_allclose(s.cpu().numpy(), allact.sum(0), rtol=1e-12)
  np.testing.assert_allclose(sxx.cpu().numpy(), allact.T @ allact, rtol=1e-11, atol=1e-9)
  from compare_gan_b200.metrics import fid_score
  real = rng.randn(400, d).astype(np.float32) * 1.5
  mu, sigma = fid_score.moments_from_sums(s.cpu().numpy(), sxx.cpu().numpy(), 2 * n)
  mur, sr = real.astype(np.float64).mean(0), np.cov(real.astype(np.float64), rowvar=False)
  got = fid_score.fid_from_moments(mur, sr, mu, sigma)
  ref = ometrics.compute_fid_from_activations(real, allact)
  assert abs(got - ref) <= 5e-3 * abs(ref), (got, ref)


TC_CASES = [
    # n, h, cin, cout, k, upsample      (shapes the tensor-core path accepts: cin%32==0, cout%32==0, 128-pixel boxes)
    (2, 8, 32, 32, 3, False),
    (2, 8, 64, 128, 3, False),
    (8, 4, 64, 64, 3, False),
    (2, 16, 32, 256, 3, False),
    (1, 32, 96, 192, 3, False),
    (4, 8, 64, 64, 1, False),
    (2, 8, 64, 32, 3, True),
    (1, 32, 256, 256, 3, False),
    (1, 64, 32, 96, 3, False),
    (2, 16, 384, 512, 3, False),
    (2, 8, 128, 64, 3, False),
    (2, 8, 128, 128, 3, True),
    (8, 4, 256, 96, 3, True),
    (4, 8, 128, 32, 1, False),
    (1, 64, 128, 128, 3, False),
    (2, 16, 64, 3, 3, False),      # thin image conv: Cout=3 zero-padded to a 32-column tile
    (2, 8, 32, 20, 1, False),
    (2, 16, 96, 192, 3, False),    # Cin not a multiple of 128: zero-padded ci tile in the tensor-core wgrad
    (2, 8, 192, 96, 3, True),
    (3, 35, 48, 64, 5, False),     # Inception-A: 35x35 map (105-row boxes), 25 taps, K=48 zero-padded to 64
    (2, 17, 128, 192, 7, False),   # 17x17 map; square 7x7 here (49 taps) falls back to the gather-GEMM
    (5, 8, 80, 96, 3, False),      # 8x8 maps, odd batch: the last tile hangs over the batch
    (1, 147, 32, 64, 3, False),    # 147-wide rows split into two 74-pixel boxes
    (8, 4, 32, 64, 1, True),       # 1x1 over a zero-inserted input: phase (0,0) on the tensor cores + bias-only phases
    (2, 16, 192, 96, 1, True),
]


@pytest.mark.parametrize("n,h,cin,cout,k", [(2, 16, 64, 128, 4), (8, 8, 128, 256, 4), (2, 32, 64, 64, 3), (1, 64, 128, 128, 4)])
def test_conv2d_stride2_tcgen05(K, n, h, cin, cout, k):
  """Stride-2 convs (SNDCGAN D 4x4 s2, and its generator's transposed convs = their input gradient) on the tensor cores through
  the four parity-phase TMA views."""
  rng = np.random.RandomState(n * 100 + h + cin + k)
  x = rng.randn(n, h, h, cin).astype(np.float32)
  w = (rng.randn(k, k, cin, cout) / np.sqrt(k * k * cin)).astype(np.float32)
  b = rng.randn(cout).astype(np.float32)
  xt, wt = torch.from_numpy(x).requires_grad_(True), torch.from_numpy(w).requires_grad_(True)
  ref = T.conv2d_same(xt, wt, 2) + torch.from_numpy(b)
  gy = rng.randn(*ref.shape).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  K.set_math_mode(1)
  try:
    xd, wd, bd = dev(K, x, True), dev(K, w, True), dev(K, b, True)
    n0 = K.lib().launch_count()
    y = K.conv2d(xd, wd, bd, stride=2)
    assert K.lib().launch_count() - n0 == 2, "expected weight prep + one tensor-core launch"
    assert_close(y.cpu(), ref.detach().numpy(), 1e-3, "s2 fwd")
    gx, gw = tape_grads(K, y, gy, [xd, wd])
    assert_close(gx.cpu(), xt.grad.numpy(), 1e-3, "s2 dgrad")
    assert_close(gw.cpu(), wt.grad.numpy(), 1e-3, "s2 wgrad")
  finally:
    K.set_math_mode(0)


@pytest.mark.parametrize("n,h,cin,cout,k,up", TC_CASES)
def test_conv2d_tcgen05_tf32(K, n, h, cin, cout, k, up):
  """math_mode 1: wgmma TF32 implicit GEMM (TMA-staged, register accumulators) vs the fp32 oracle.
  Tolerance 1e-3 rel-L2 (north_star's per-tensor bound); expected ~3e-4 for RN-rounded TF32 operands."""
  rng = np.random.RandomState(hash((n, h, cin, cout, k, up)) % 2**31)
  x = rng.randn(n, h, h, cin).astype(np.float32)
  w = (rng.randn(k, k, cin, cout) / np.sqrt(k * k * cin)).astype(np.float32)
  b = rng.randn(cout).astype(np.float32)
  xt = torch.from_numpy(x).requires_grad_(True)
  wt = torch.from_numpy(w).requires_grad_(True)
  ref = T.conv2d_same(T.unpool(xt) if up else xt, wt, 1) + torch.from_numpy(b)
  gy = rng.randn(*ref.shape).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  K.set_math_mode(1)
  try:
    xd, wd, bd = dev(K, x, True), dev(K, w, True), dev(K, b, True)
    n0 = K.lib().launch_count()
    y = K.conv2d(xd, wd, bd, stride=1, upsample=up)
    launched = K.lib().launch_count() - n0
    if k == 1 and up:
      assert launched == 3, "1x1 up-sampling conv: weight prep + one tensor-core phase + bias fill, got %d" % launched
    elif min(cin, cout) <= 4 and not up:
      # image-side layer (csrc/thin_tc.cu): filter re-layout + weight prep + ONE 32-wide tensor-core GEMM + the shift-add pass
      assert launched == 4, "expected the patch-tensor tensor-core path (4 launches), got %d" % launched
    elif k * k <= 32:
      # (the four sub-pixel phases of a convolution over a zero-inserted input share one weight preparation and ONE launch)
      assert launched == 2, "expected the tensor-core path (weight prep + one launch), got %d launches" % launched
    assert_close(y.cpu(), ref.detach().numpy(), 1e-3, "tc conv fwd")
    gx, gw = tape_grads(K, y, gy, [xd, wd])
    assert_close(gx.cpu(), xt.grad.numpy(), 1e-3, "tc conv dgrad")
    assert_close(gw.cpu(), wt.grad.numpy(), 1e-3, "wgrad")
  finally:
    K.set_math_mode(0)
  # unbiasedness of the rounding (truncation would shift the mean ratio by ~ -5e-4)
  yy, rr = y.cpu().astype(np.float64).ravel(), ref.detach().numpy().astype(np.float64).ravel()
  ratio = float((yy * rr).sum() / (rr * rr).sum())
  assert abs(ratio - 1.0) < 1.5e-4, ratio


@pytest.mark.parametrize("n,h,cin,cout,k", [(2, 35, 64, 96, 3), (1, 71, 80, 192, 3), (3, 8, 32, 64, 5)])
def test_conv2d_valid_padding_tcgen05(K, n, h, cin, cout, k):
  """VALID (unpadded) stride-1 convolutions (Inception stem) on the tensor cores: the tile grid is the smaller output extent."""
  import torch.nn.functional as F
  rng = np.random.RandomState(h + cin)
  x = rng.randn(n, h, h, cin).astype(np.float32)
  w = (rng.randn(k, k, cin, cout) / np.sqrt(k * k * cin)).astype(np.float32)
  b = rng.randn(cout).astype(np.float32)
  ref = F.conv2d(torch.from_numpy(x).permute(0, 3, 1, 2), torch.from_numpy(w).permute(3, 2, 0, 1)).permute(0, 2, 3, 1) + torch.from_numpy(b)
  for mode, tol in ((0, 2e-5), (1, 1e-3)):
    K.set_math_mode(mode)
    try:
      n0 = K.lib().launch_count()
      y = K.conv2d(dev(K, x), dev(K, w), dev(K, b), padding="VALID")
      if mode == 1:
        assert K.lib().launch_count() - n0 == 2
      yr = K.conv2d_relu(dev(K, x), dev(K, w), dev(K, b), padding="VALID")
    finally:
      K.set_math_mode(0)
    assert y.shape == tuple(ref.shape)
    assert_close(y.cpu(), ref.numpy(), tol, "valid conv mode %d" % mode)
    assert_close(yr.cpu(), torch.relu(ref).numpy(), tol * 2, "valid conv+relu mode %d" % mode)


@pytest.mark.parametrize("n,h,cin,cout,k,pad", [(2, 17, 192, 320, 3, "VALID"), (2, 35, 288, 384, 3, "VALID"),
                                                 (2, 9, 64, 64, 3, "SAME"), (3, 299, 3, 32, 3, "VALID")])
def test_conv2d_stride2_any_size_tcgen05(K, n, h, cin, cout, k, pad):
  """Stride-2 convs on odd-sized maps, SAME or VALID (Inception's reductions 35->17->8): the four parity phases have
  different extents, each gets its own TMA view."""
  import torch.nn.functional as F
  rng = np.random.RandomState(h + cin)
  x = rng.randn(n, h, h, cin).astype(np.float32)
  w = (rng.randn(k, k, cin, cout) / np.sqrt(k * k * cin)).astype(np.float32)
  b = rng.randn(cout).astype(np.float32)
  if pad == "SAME":
    ref = T.conv2d_same(torch.from_numpy(x), torch.from_numpy(w), 2) + torch.from_numpy(b)
  else:
    ref = F.conv2d(torch.from_numpy(x).permute(0, 3, 1, 2), torch.from_numpy(w).permute(3, 2, 0, 1), stride=2).permute(0, 2, 3, 1) + torch.from_numpy(b)
  K.set_math_mode(1)
  try:
    n0 = K.lib().launch_count()
    y = K.conv2d_relu(dev(K, x), dev(K, w), dev(K, b), stride=2, padding=pad)
    launched = K.lib().launch_count() - n0
  finally:
    K.set_math_mode(0)
  if cin % 4 == 0:
    assert launched == 2, "expected the tensor-core path"
  assert y.shape == tuple(ref.shape)
  assert_close(y.cpu(), torch.relu(ref).numpy(), 1e-3, "stride-2 %s conv" % pad)


@pytest.mark.parametrize("rows,cols", [(70, 1024), (33, 256), (5, 100)])
def test_softmax_rows(K, rows, cols):
  rng = np.random.RandomState(cols)
  x = (rng.randn(rows, cols) * 3).astype(np.float32)
  gy = rng.randn(rows, cols).astype(np.float32)
  xt = torch.from_numpy(x).requires_grad_(True)
  ref = torch.softmax(xt, -1)
  ref.backward(torch.from_numpy(gy))
  xd = dev(K, x, True)
  y = K.softmax(xd)
  assert_close(y.cpu(), ref.detach().numpy(), 1e-6, "softmax")
  (gx,) = tape_grads(K, y, gy, [xd])
  assert_close(gx.cpu(), xt.grad.numpy(), 2e-5, "softmax grad")


@pytest.mark.parametrize("bsz,m,kv,ca,cg", [(3, 1024, 256, 24, 96), (2, 4096, 1024, 12, 48), (5, 256, 64, 32, 64)])
def test_tc_batched_matmul_attention(K, bsz, m, kv, ca, cg):
  """math_mode 1: the attention products of the non-local block (arch_ops.py:744, 753) and all four of their
  gradients run as per-image GEMMs on the tensor cores: nt / nn through the conv kernel (per-image weight slice), tn through
  the filter-gradient kernel (one image per CTA row)."""
  rng = np.random.RandomState(m + kv)
  theta = rng.randn(bsz, m, ca).astype(np.float32)
  phi = rng.randn(bsz, kv, ca).astype(np.float32)
  g = rng.randn(bsz, kv, cg).astype(np.float32)
  tt, pt, gt = [torch.from_numpy(a).requires_grad_(True) for a in (theta, phi, g)]
  logits = torch.bmm(tt, pt.transpose(1, 2)) / np.sqrt(ca)
  ref = torch.bmm(logits, gt)
  gy = rng.randn(*ref.shape).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  K.set_math_mode(1)
  try:
    td, pd, gd = dev(K, theta, True), dev(K, phi, True), dev(K, g, True)
    n0 = K.lib().launch_count()
    s = K.affine(K.bmm(td, pd, False, True), 1.0 / np.sqrt(ca))
    y = K.bmm(s, gd)
    assert K.lib().launch_count() - n0 == 5, "expected 2 x (operand prep + tensor-core launch) + scale"
    assert_close(y.cpu(), ref.detach().numpy(), 2e-3, "attn fwd")
    n0 = K.lib().launch_count()
    gth, gph, gg = tape_grads(K, y, gy, [td, pd, gd])
    assert_close(gth.cpu(), tt.grad.numpy(), 2e-3, "d theta (nn)")
    assert_close(gph.cpu(), pt.grad.numpy(), 2e-3, "d phi (tn)")
    assert_close(gg.cpu(), gt.grad.numpy(), 2e-3, "d g (tn)")
  finally:
    K.set_math_mode(0)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("n,h,cin,cout,k,stride,pad", [(64, 8, 64, 96, 3, 1, "SAME"), (8, 17, 32, 64, 3, 2, "VALID"),
                                                       (4, 35, 48, 64, 5, 1, "SAME"), (64, 8, 128, 320, 1, 1, "SAME"),
                                                       (4, 35, 3, 32, 3, 2, "VALID"), (16, 32, 3, 128, 3, 1, "SAME")])
def test_conv_into_channel_slice(K, mode, n, h, cin, cout, k, stride, pad):
  """cgan_conv2d_fwd_act_ld: the convolution stores into its channel slice of a wider NHWC tensor (the Inception
  concat without the copy); the neighbouring channels stay untouched.  The 8x8 cases also take the narrow column tiles
  the occupancy rule picks when there are fewer pixel tiles than SMs; the 3-channel cases run the thin-Cin kernel."""
  rng = np.random.RandomState(n + h + cin)
  x = rng.randn(n, h, h, cin).astype(np.float32)
  w = (rng.randn(k, k, cin, cout) / np.sqrt(k * k * cin)).astype(np.float32)
  b = rng.randn(cout).astype(np.float32)
  xt = torch.from_numpy(x).permute(0, 3, 1, 2)
  if pad == "SAME":
    ref = T.conv2d_same(torch.from_numpy(x), torch.from_numpy(w), stride) + torch.from_numpy(b)
  else:
    ref = F.conv2d(xt, torch.from_numpy(w).permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1) + torch.from_numpy(b)
  ref = torch.relu(ref).numpy()
  K.set_math_mode(mode)
  try:
    sink = K.ChannelSink(cout + 40)
    buf = sink.buffer(n, ref.shape[1], ref.shape[2])
    K.fill_(buf, 7.0)
    assert K.conv2d_relu(dev(K, x), dev(K, w), dev(K, b), stride=stride, padding=pad, sink=sink, sink_off=24) is None
    whole = K.conv2d_relu(dev(K, x), dev(K, w), dev(K, b), stride=stride, padding=pad).cpu()
  finally:
    K.set_math_mode(0)
  out = buf.cpu()
  assert_close(out[..., 24:24 + cout], ref, 1e-3 if mode else TOL, "sliced conv")
  np.testing.assert_array_equal(out[..., 24:24 + cout], whole)       # same kernel, same K order: bit-identical
  assert (out[..., :24] == 7.0).all() and (out[..., 24 + cout:] == 7.0).all()


def _rna_tf32(a):
  a = np.ascontiguousarray(a, np.float32)
  return ((a.view(np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


@pytest.mark.parametrize("bsz,lq,lk,dk,dv", [(3, 256, 128, 24, 96), (2, 1024, 256, 12, 48), (2, 4096, 1024, 24, 96),
                                              (2, 4096, 1024, 12, 48), (1, 128, 128, 32, 128), (2, 256, 128, 4, 16)])
def test_tc_fused_attention(K, bsz, lq, lk, dk, dv):
  """math_mode 1: softmax(theta phi^T) g of the non-local block (arch_ops.py:744-753) and its three gradients in the fused
  wgmma kernels (csrc/attn_tc.cu) — scores only in registers.  Checked (a) against the float64 evaluation on the
  SAME TF32-rounded operands (what remains is the TF32 rounding of the probabilities and fp32 accumulation: <= 5e-4), (b) against
  the reference's own composition tf.matmul -> tf.nn.softmax -> tf.matmul in fp32 on the unrounded operands at north_star's
  1e-3, and (c) against the engine's composed path (three launches per direction) in exact-fp32 mode."""
  rng = np.random.RandomState(lq + lk + dk)
  theta = (0.5 * rng.randn(bsz, lq, dk)).astype(np.float32)
  phi = (0.5 * rng.randn(bsz, lk, dk)).astype(np.float32)
  g = rng.randn(bsz, lk, dv).astype(np.float32)
  gy = rng.randn(bsz, lq, dv).astype(np.float32)

  def torch_ref(arrs, dtype):
    tt, pt, gt = [torch.from_numpy(a).to(dtype).requires_grad_(True) for a in arrs[:3]]
    out = torch.bmm(torch.softmax(torch.bmm(tt, pt.transpose(1, 2)), -1), gt)
    out.backward(torch.from_numpy(arrs[3]).to(dtype))
    return [t.detach().numpy() for t in (out, tt.grad, pt.grad, gt.grad)]
  ref32 = torch_ref((theta, phi, g, gy), torch.float32)
  ref64 = torch_ref((_rna_tf32(theta), _rna_tf32(phi), _rna_tf32(g), _rna_tf32(gy)), torch.float64)

  K.set_math_mode(1)
  try:
    assert K.attention_shape_ok(bsz, lq, lk, dk, dv)
    td, pd, gd = dev(K, theta, True), dev(K, phi, True), dev(K, g, True)
    n0 = K.lib().launch_count()
    y = K.attention(td, pd, gd)
    assert K.lib().launch_count() - n0 == 4, "3 operand roundings + ONE fused forward kernel"
    n0 = K.lib().launch_count()
    grads = tape_grads(K, y, gy, [td, pd, gd])
    assert K.lib().launch_count() - n0 <= 5, "rounding of dO + rowdot + the dQ kernel + the dK/dV kernel"
    got = [y.cpu()] + [t.cpu() for t in grads]
  finally:
    K.set_math_mode(0)
  for name, a, r64, r32 in zip(("out", "d theta", "d phi", "d g"), got, ref64, ref32):
    assert_close(a, r64, 5e-4, "fused attention %s vs float64 on the TF32-rounded operands" % name)
    assert_close(a, r32, 1e-3, "fused attention %s vs fp32 reference composition" % name)
  # the composed path (exact fp32) of the same op
  td, pd, gd = dev(K, theta, True), dev(K, phi, True), dev(K, g, True)
  y0 = K.attention(td, pd, gd)
  grads0 = tape_grads(K, y0, gy, [td, pd, gd])
  for name, a, b in zip(("out", "d theta", "d phi", "d g"), got, [y0.cpu()] + [t.cpu() for t in grads0]):
    assert_close(a, b, 1e-3, "fused vs composed attention %s" % name)


def test_attention_falls_back_for_shapes_the_fused_kernel_does_not_take(K):
  """Toy widths (2 key channels at ch = 8) and math_mode 0 compose bmm -> softmax -> bmm like the reference."""
  rng = np.random.RandomState(5)
  theta, phi, g = rng.randn(2, 64, 2).astype(np.float32), rng.randn(2, 16, 2).astype(np.float32), rng.randn(2, 16, 8).astype(np.float32)
  ref = torch.bmm(torch.softmax(torch.bmm(torch.from_numpy(theta), torch.from_numpy(phi).transpose(1, 2)), -1), torch.from_numpy(g))
  for mode in (0, 1):
    K.set_math_mode(mode)
    try:
      assert not K.attention_shape_ok(2, 64, 16, 2, 8)
      y = K.attention(dev(K, theta), dev(K, phi), dev(K, g))
    finally:
      K.set_math_mode(0)
    assert_close(y.cpu(), ref.numpy(), 1e-3 if mode else TOL, "composed attention")
  assert not K.attention_shape_ok(2, 4096, 1024, 24, 96), "math_mode 0 never takes the TF32 kernel"


THIN_TC_CASES = [
    # n, h, cin, cout, k, stride, padding          image-side layers of the BASELINE architectures
    (8, 32, 3, 128, 3, 1, "SAME"),     # resnet_cifar / sndcgan D: first conv
    (4, 64, 3, 96, 3, 1, "SAME"),      # BigGAN D block 1 conv1 (ch = 96)
    (4, 32, 256, 3, 3, 1, "SAME"),     # resnet_cifar G: image conv
    (2, 64, 96, 3, 3, 1, "SAME"),      # BigGAN G: image conv
    (2, 75, 3, 32, 3, 2, "VALID"),     # Inception-v3 stem (299 -> 149 at full size): stride 2, VALID
    (3, 16, 1, 64, 5, 1, "SAME"),      # one input channel, 25 taps
    (2, 32, 64, 4, 3, 1, "SAME"),      # four output channels: 36 > 32 values per pixel -> stays on the streaming kernels
]


@pytest.mark.parametrize("n,h,cin,cout,k,stride,pad", THIN_TC_CASES)
def test_thin_convolutions_on_tensor_cores(K, n, h, cin, cout, k, stride, pad):
  """math_mode 1: convolutions with <= 4 input or output channels run as one 32-wide tensor-core GEMM over a [pixels, 32] patch
  tensor (csrc/thin_tc.cu) — forward, input gradient and filter gradient against the fp32 oracle at north_star's 1e-3, and
  against the exact-fp32 streaming kernels they replace (CGAN_OPT_TC_THIN = 0)."""
  from compare_gan_b200 import _lib
  rng = np.random.RandomState(n + h + cin + cout)
  x = rng.randn(n, h, h, cin).astype(np.float32)
  w = (rng.randn(k, k, cin, cout) / np.sqrt(k * k * cin)).astype(np.float32)
  b = rng.randn(cout).astype(np.float32)
  xt, wt = torch.from_numpy(x).requires_grad_(True), torch.from_numpy(w).requires_grad_(True)
  if pad == "SAME":
    ref = T.conv2d_same(xt, wt, stride) + torch.from_numpy(b)
  else:
    ref = F.conv2d(xt.permute(0, 3, 1, 2), wt.permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1) + torch.from_numpy(b)
  gy = rng.randn(*ref.shape).astype(np.float32)
  ref.backward(torch.from_numpy(gy))
  refs = [ref.detach().numpy(), xt.grad.numpy(), wt.grad.numpy()]
  expect_tc = k * k * min(cin, cout) <= 32
  lib = K.lib()
  results = {}
  K.set_math_mode(1)
  try:
    for thin in (1, 0):
      lib.set_option(_lib.OPT_TC_THIN, thin)
      xd, wd, bd = dev(K, x, True), dev(K, w, True), dev(K, b, True)
      y = K.conv2d(xd, wd, bd, stride=stride, padding=pad)
      path = _lib.PATH_NAMES[lib.get_option(_lib.OPT_LAST_PATH)]
      gx, gw = tape_grads(K, y, gy, [xd, wd])
      results[thin] = ([y.cpu(), gx.cpu(), gw.cpu()], path)
  finally:
    lib.set_option(_lib.OPT_TC_THIN, 1)
    K.set_math_mode(0)
  if not getattr(lib, "emulated", False):
    assert results[1][1] == ("tcgen05_tf32" if expect_tc else results[0][1]), results[1][1]
    assert results[0][1] != "tcgen05_tf32" or min(cin, cout) > 4 or cout <= 4, results[0][1]
  for name, a, a0, r in zip(("fwd", "dgrad", "wgrad"), results[1][0], results[0][0], refs):
    assert_close(a, r, 1e-3, "thin-tc %s vs fp32 oracle" % name)
    assert_close(a, a0, 1e-3, "thin-tc %s vs streaming kernels" % name)


def test_random_uniform_is_the_documented_counter_based_stream(K):
  """cgan_random_uniform (the un-fed WGAN-GP interpolation coefficients, penalty_lib.py:72-73): SplitMix64(seed, offset + i),
  top 24 bits -> [0, 1); stateless, so two launches over adjacent ranges continue one stream."""
  n, seed = 4099, 0x5EEDA1FA
  out = K.empty(n)
  K._call("random_uniform", out.ptr, 1000, seed, 7)
  K._call("random_uniform", out.ptr + 4 * 1000, n - 1000, seed, 1007)
  got = out.cpu()
  idx = np.arange(1, n + 1, dtype=np.uint64) + np.uint64(7)
  with np.errstate(over="ignore"):
    z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * idx
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
  ref = (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
  np.testing.assert_array_equal(got, ref)
  assert 0.0 <= got.min() and got.max() < 1.0 and abs(got.mean() - 0.5) < 0.02
