"""Oracle (test infrastructure): TF1 op semantics restated on PyTorch-CPU fp32.

All activations are NHWC ``torch.float32`` tensors; conv kernels are HWIO
``[kh,kw,cin,cout]``; deconv kernels ``[kh,kw,cout,cin]``; linear kernels
``[in,out]`` — exactly the reference layouts (architectures/arch_ops.py:543-546,
563-565, 583-585).  Backward passes come from torch.autograd (an independent
implementation from the hand-written CUDA backward under test).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


def _same_pads(n, k, s):
  """TF SAME padding (SURVEY App. A): out=ceil(n/s); before=total//2."""
  out = -(-n // s)
  total = max((out - 1) * s + k - n, 0)
  return out, total // 2, total - total // 2


# ---------------------------------------------------------------------------------------------------------------------
# TF32-operand emulation (test infrastructure).  The engine's math_mode 1 evaluates every convolution-like contraction
# that the library routes to the tensor cores as: round both operands to the nearest TF32 value (cvt.rna: 10 mantissa
# bits, ties away from zero), multiply exactly, accumulate in fp32.  Its backward applies the same rule to each gradient
# contraction separately (dx = dgrad(rna(dy), rna(w)), dw = wgrad(rna(x), rna(dy))).  With TF32_PLAN set to the
# {(kind, n, h, w, cin, cout, kh, kw, stride): path} dictionary recorded by the engine (kernels.CONV_TRACE), the
# convolutions below reproduce exactly that arithmetic, so an engine run in math_mode 1 can be compared with this oracle
# at fp32-accumulation-order tolerance (~1e-5) instead of the ~1e-3 that separates TF32 from fp32 — and the difference
# between this oracle with and without the plan is what the precision mode itself costs, independent of our kernels.
TF32_PLAN = None


def rna_tf32(t):
  """Round to the nearest TF32-representable value, ties away from zero (PTX cvt.rna.tf32.f32)."""
  a = t.detach().to(torch.float32).contiguous()
  bits = a.view(torch.int32)
  out = ((bits + 0x1000) & ~0x1FFF).view(torch.float32)
  return out.to(t.dtype)


def _tf32_used(kind, key):
  """(first operand rounded, second operand rounded) for this contraction, from the engine's record."""
  if TF32_PLAN is None:
    return False, False
  rec = TF32_PLAN.get((kind,) + tuple(int(v) for v in key))
  if rec is None and kind == "bmm" and any(k[0] == "attention" and k[1] == int(key[0]) for k in TF32_PLAN):
    # the engine ran this block's products inside its fused attention kernels (kernels.attention): every operand of the
    # five products (theta, phi, g, the probabilities, dS, d out) enters them rounded to TF32
    return True, True
  if rec is None:
    raise KeyError("TF32 plan has no entry for %s %s (the engine never ran this contraction)" % (kind, key))
  return bool(rec[1]), bool(rec[2])


def _r(t, on):
  return rna_tf32(t) if on else t


def _conv_key(x_shape, w_shape, stride):
  n, h, w, cin = x_shape
  kh, kw, _, cout = w_shape
  return (n, h, w, cin, cout, kh, kw, stride)


def _conv_raw(x, w_hwio, stride):
  kh, kw = w_hwio.shape[0], w_hwio.shape[1]
  _, pt, pb = _same_pads(x.shape[1], kh, stride)
  _, pl, pr = _same_pads(x.shape[2], kw, stride)
  xn = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
  return F.conv2d(xn, w_hwio.permute(3, 2, 0, 1), stride=stride).permute(0, 2, 3, 1)


def _dgrad_raw(gy, w_hwio, x_shape, stride):
  kh, kw = w_hwio.shape[0], w_hwio.shape[1]
  n, h, w, cin = x_shape
  _, pt, pb = _same_pads(h, kh, stride)
  _, pl, pr = _same_pads(w, kw, stride)
  gxp = torch.nn.grad.conv2d_input((n, cin, h + pt + pb, w + pl + pr), w_hwio.permute(3, 2, 0, 1),
                                   gy.permute(0, 3, 1, 2), stride=stride)
  return gxp[:, :, pt:pt + h, pl:pl + w].permute(0, 2, 3, 1)


def _wgrad_raw(x, gy, w_shape, stride):
  kh, kw, cin, cout = w_shape
  _, pt, pb = _same_pads(x.shape[1], kh, stride)
  _, pl, pr = _same_pads(x.shape[2], kw, stride)
  xn = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
  gw = torch.nn.grad.conv2d_weight(xn, (cout, cin, kh, kw), gy.permute(0, 3, 1, 2), stride=stride)
  return gw.permute(2, 3, 1, 0)


class _Tf32Conv(torch.autograd.Function):
  """y = conv(x, w) with the engine's per-contraction operand rounding; mirrors kernels.conv2d / _taped_fwd."""

  @staticmethod
  def forward(ctx, x, w, stride):
    ctx.save_for_backward(x, w)
    ctx.stride = stride
    ra, rb = _tf32_used("fwd", _conv_key(x.shape, w.shape, stride))
    return _conv_raw(_r(x, ra), _r(w, rb), stride)

  @staticmethod
  def backward(ctx, gy):
    x, w = ctx.saved_tensors
    gx = _Tf32Dgrad.apply(gy, w, tuple(x.shape), ctx.stride) if ctx.needs_input_grad[0] else None
    gw = _Tf32Wgrad.apply(x, gy, tuple(w.shape), ctx.stride) if ctx.needs_input_grad[1] else None
    return gx, gw, None


class _Tf32Dgrad(torch.autograd.Function):
  """dx = conv_transpose(dy, w); mirrors kernels.conv2d_dgrad (linear in dy and in w)."""

  @staticmethod
  def forward(ctx, gy, w, x_shape, stride):
    ctx.save_for_backward(gy, w)
    ctx.x_shape, ctx.stride = x_shape, stride
    ra, rb = _tf32_used("dgrad", _conv_key(x_shape, w.shape, stride))
    return _dgrad_raw(_r(gy, ra), _r(w, rb), x_shape, stride)

  @staticmethod
  def backward(ctx, ggx):
    gy, w = ctx.saved_tensors
    ggy = _Tf32Conv.apply(ggx, w, ctx.stride) if ctx.needs_input_grad[0] else None
    gw = _Tf32Wgrad.apply(ggx, gy, tuple(w.shape), ctx.stride) if ctx.needs_input_grad[1] else None
    return ggy, gw, None, None


class _Tf32Wgrad(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, gy, w_shape, stride):
    ra, rb = _tf32_used("wgrad", _conv_key(x.shape, w_shape, stride))
    return _wgrad_raw(_r(x, ra), _r(gy, rb), w_shape, stride)

  @staticmethod
  def backward(ctx, g):
    raise NotImplementedError("third-order differentiation through the filter gradient is not needed on this path")


class _Tf32Bmm(torch.autograd.Function):
  """op(a) @ op(b) per image with the engine's operand rounding (kernels.bmm: attention products, arch_ops.py:744,753)."""

  @staticmethod
  def forward(ctx, a, b, ta, tb):
    ctx.save_for_backward(a, b)
    ctx.ta, ctx.tb = ta, tb
    return _bmm_raw(a, b, ta, tb)

  @staticmethod
  def backward(ctx, g):
    a, b = ctx.saved_tensors
    ta, tb = ctx.ta, ctx.tb
    ga = gb = None
    if ctx.needs_input_grad[0]:
      ga = _bmm_raw(b, g, tb, True) if ta else _bmm_raw(g, b, False, not tb)
    if ctx.needs_input_grad[1]:
      gb = _bmm_raw(g, a, True, ta) if tb else _bmm_raw(a, g, not ta, False)
    return ga, gb, None, None


def _bmm_raw(a, b, ta, tb):
  bsz = a.shape[0]
  m = a.shape[2] if ta else a.shape[1]
  k = a.shape[1] if ta else a.shape[2]
  n = b.shape[1] if tb else b.shape[2]
  ra, rb = _tf32_used("bmm", (bsz, int(ta), int(tb), m, n, k))
  a, b = _r(a, ra), _r(b, rb)
  return torch.bmm(a.transpose(1, 2) if ta else a, b.transpose(1, 2) if tb else b)


def bmm(a, b, ta=False, tb=False):
  """Batched tf.matmul (arch_ops.py:744, 753); follows the TF32 plan when one is set."""
  if TF32_PLAN is None:
    return torch.bmm(a.transpose(1, 2) if ta else a, b.transpose(1, 2) if tb else b)
  return _Tf32Bmm.apply(a, b, ta, tb)


def conv2d_same(x, w_hwio, stride=1):
  """tf.nn.conv2d(x, w, strides=[1,s,s,1], padding="SAME") — arch_ops.py:568."""
  if TF32_PLAN is not None:
    return _Tf32Conv.apply(x, w_hwio, stride)
  kh, kw = w_hwio.shape[0], w_hwio.shape[1]
  _, pt, pb = _same_pads(x.shape[1], kh, stride)
  _, pl, pr = _same_pads(x.shape[2], kw, stride)
  xn = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb))
  y = F.conv2d(xn, w_hwio.permute(3, 2, 0, 1), stride=stride)
  return y.permute(0, 2, 3, 1)


def conv2d_transpose_same(x, w_hwoi, out_hw, stride):
  """tf.nn.conv2d_transpose (default SAME) — arch_ops.py:588-589.

  Adjoint of "SAME-pad then VALID conv": full transposed conv, then crop the
  SAME padding.  ``w_hwoi`` is ``[kh,kw,cout,cin]`` (cin = x channels).
  """
  if TF32_PLAN is not None:
    # w is the HWIO kernel of the conv that maps the OUTPUT (cout channels) back to x: deconv(x) is its input gradient
    n = x.shape[0]
    return _Tf32Dgrad.apply(x, w_hwoi, (n, out_hw[0], out_hw[1], w_hwoi.shape[2]), stride)
  kh, kw = w_hwoi.shape[0], w_hwoi.shape[1]
  oh, ow = out_hw
  _, pt, _ = _same_pads(oh, kh, stride)
  _, pl, _ = _same_pads(ow, kw, stride)
  # torch conv_transpose2d weight: [in_channels(=cin of x), out_channels, kh, kw]
  wt = w_hwoi.permute(3, 2, 0, 1)
  full = F.conv_transpose2d(x.permute(0, 3, 1, 2), wt, stride=stride)
  need_h, need_w = pt + oh, pl + ow
  if full.shape[2] < need_h or full.shape[3] < need_w:
    full = F.pad(full, (0, max(0, need_w - full.shape[3]),
                        0, max(0, need_h - full.shape[2])))
  y = full[:, :, pt:pt + oh, pl:pl + ow]
  return y.permute(0, 2, 3, 1)


def unpool(x):
  """Zero-insertion 2x upsampling — resnet_ops.py:35-56 (value at even r,c)."""
  n, h, w, c = x.shape
  out = torch.zeros(n, 2 * h, 2 * w, c, dtype=x.dtype)
  out[:, ::2, ::2, :] = x
  return out


def avg_pool2(x):
  """tf.nn.pool(x,[2,2],"AVG","SAME",strides=[2,2]) — resnet_ops.py:131-133."""
  return F.avg_pool2d(x.permute(0, 3, 1, 2), 2, 2, ceil_mode=True,
                      count_include_pad=False).permute(0, 2, 3, 1)


def max_pool2(x):
  """tf.layers.max_pooling2d(pool 2, stride 2, VALID) — arch_ops.py:741,750."""
  return F.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)


def lrelu(x, leak=0.2):
  """arch_ops.py:595-597: max(x, leak*x), with the gradient of TF's Maximum: 1 where x >= 0 (a tie, x = +-0, sends it to
  x), leak elsewhere.  torch.maximum would split a tie's gradient between its arguments."""
  return torch.where(x >= 0, x, leak * x)


def l2_normalize(x, eps=1e-12):
  """tf.math.l2_normalize over all elements: x*rsqrt(max(sum x^2, eps))."""
  return x * torch.rsqrt(torch.clamp((x * x).sum(), min=eps))


def batch_moments(x4):
  """arch_ops.py:289-297: fp32 mean and BIASED variance, E[x^2]-E[x]^2 form."""
  mean = x4.mean(dim=(0, 1, 2))
  mean_sq = (x4 * x4).mean(dim=(0, 1, 2))
  return mean, mean_sq - mean * mean


def cross_replica_mean(shards):
  """tpu/tpu_ops.py:75-91: sum over replicas / group size (list of tensors)."""
  tot = shards[0].clone()
  for s in shards[1:]:
    tot = tot + s
  return tot / float(len(shards))


def cross_replica_moments(shards4):
  """tpu/tpu_ops.py:94-125 with parallel=True: mean of per-replica means and of
  per-replica mean-of-squares; var = E[x^2] - E[x]^2."""
  means = [s.mean(dim=(0, 1, 2)) for s in shards4]
  msqs = [(s * s).mean(dim=(0, 1, 2)) for s in shards4]
  mean = cross_replica_mean(means)
  msq = cross_replica_mean(msqs)
  return mean, msq - mean * mean


def normalize(x4, mean, var, eps):
  """tf.nn.batch_normalization with scale/offset None — arch_ops.py:306-312."""
  inv = torch.rsqrt(var + eps)
  return x4 * inv + (-mean * inv)


def spectral_sigma(w2d, u, singular_value="left", eps=1e-12):
  """One power iteration — arch_ops.py:503-527.  Returns (sigma, u_new, v).

  u_new and v are detached (stop_gradient, :521-522); sigma keeps grad wrt w.
  """
  with torch.no_grad():
    if singular_value == "left":
      v = l2_normalize(w2d.t() @ u, eps)
      u_new = l2_normalize(w2d @ v, eps)
    else:
      v = l2_normalize(u @ w2d.t(), eps)
      u_new = l2_normalize(v @ w2d, eps)
  if singular_value == "left":
    sigma = (u_new.t() @ w2d) @ v
  else:
    sigma = (v @ w2d) @ u_new.t()
  return sigma.reshape(()), u_new, v


def sigmoid_ce(logits, labels_one):
  """tf.nn.sigmoid_cross_entropy_with_logits: max(x,0)-x*z+log1p(exp(-|x|)), written as TF writes it (x >= 0 selects both
  branches), so that its gradient is sigmoid(x) - z at x = 0 too (torch's clamp and abs would give 1 - z there)."""
  z = 1.0 if labels_one else 0.0
  pos = logits >= 0
  relu_logits = torch.where(pos, logits, torch.zeros_like(logits))
  neg_abs = torch.where(pos, -logits, logits)
  return relu_logits - logits * z + torch.log1p(torch.exp(neg_abs))


def orthogonal_init(rng, shape, gain=1.0):
  """tf.initializers.orthogonal (weights.initializer="orthogonal", arch_ops.py:60-61)."""
  rows = int(np.prod(shape[:-1]))
  cols = int(shape[-1])
  a = rng.standard_normal((max(rows, cols), min(rows, cols)))
  q, r = np.linalg.qr(a)
  q = q * np.sign(np.diag(r))
  if rows < cols:
    q = q.T
  return (gain * q.reshape(shape)).astype(np.float32)


def glorot_normal_init(rng, shape):
  """tf.initializers.glorot_normal: truncated normal, stddev sqrt(2/(fan_in+fan_out))
  (TF divides by .87962566103423978 to correct for truncation)."""
  fan_in, fan_out = shape[0], shape[1]
  std = math.sqrt(2.0 / (fan_in + fan_out)) / .87962566103423978
  a = rng.standard_normal(shape)
  bad = np.abs(a) > 2.0
  while bad.any():
    a[bad] = rng.standard_normal(int(bad.sum()))
    bad = np.abs(a) > 2.0
  return (a * std).astype(np.float32)
