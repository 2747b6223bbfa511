"""Taped device ops: each function launches sm_90a kernels through the C-ABI (include/cgan_b200.h)
and records its vector-Jacobian product on the tape (tape.py).  The vjps of the ops a discriminator
without normalisation is made of (convolutions, matmul, bias, (leaky) ReLU, pools, reshapes, adds) are
written with the same taped ops, so second-order differentiation (WGAN-GP, gans/penalty_lib.py:59-82)
works by construction for them.  The vjps of batch norm, softmax and spectral normalisation w.r.t. its
weight launch raw kernels: differentiating THROUGH them (a gradient penalty on a discriminator with
BN / attention) raises NotImplementedError instead of silently dropping the second-order terms.

These are the H100 stand-ins for the TF library calls the reference's ops library makes
(arch_ops.py / resnet_ops.py / loss_lib.py / penalty_lib.py); file:line citations sit on each op.
"""
import ctypes

import torch

from . import _lib
from .tape import DT, attach, no_record, recording
from .tape import grad_accumulator as _grad_accumulator, take_sink as _take_sink, sole_consumer as _sole_consumer

_RT = {"lib": None, "device": None, "math_mode": 0}

# test hook: when set to a dict, every contraction records what arithmetic it performed —
# {(kind, n, h, w, cin, cout, kh, kw, stride): (path, a_tf32, b_tf32)} with path "tcgen05_tf32" | "simt_fp32" |
# "thin_fp32", h/w the (virtual, i.e. zero-inserted) input extent, and a_tf32 / b_tf32 whether the first / second operand
# entered the products rounded to TF32 (rounded by the tensor-core kernel, or already stored rounded by its producer);
# tests feed this to the oracle's TF32-operand emulation (oracle/tf_ops.py)
CONV_TRACE = None
# test hook: callable(kind, **operands) invoked after every contraction with its operand and result tensors (tests
# recompute each one on the CPU, in situ, with the arithmetic CONV_TRACE reports)
CONV_CHECK = None


def tf32_on():
  """True in math_mode 1: tensor-core contractions round their operands to TF32, so producers may pre-round."""
  return _RT["math_mode"] == 1


def _arith(a_pre=False, b_pre=False, b_is_weight=True):
  """(path, first operand TF32-rounded, second operand TF32-rounded) of the contraction that just ran."""
  path = _lib.PATH_NAMES[_RT["lib"].get_option(_lib.OPT_LAST_PATH)]
  tc = path == "tcgen05_tf32"
  return (path, bool(tc or (a_pre and tf32_on())), bool(tc or (b_pre and tf32_on() and not b_is_weight)))


def _no_second_order(name):
  """Called by the vjps that launch raw (untaped) kernels: under tape.backward(create_graph=True) their output would
  silently lack its dependence on the incoming gradient and the stashed tensors."""
  if recording():
    raise NotImplementedError("second-order differentiation through %s is not implemented (its backward is not a taped op); "
                              "WGAN-GP style penalties need a discriminator without batch norm / attention / spectral norm "
                              "gradients in the differentiated path" % name)


def _trace(kind, key, a_pre=False, b_pre=False, b_is_weight=True):
  if CONV_TRACE is not None:
    path = _lib.PATH_NAMES[_RT["lib"].get_option(_lib.OPT_LAST_PATH)]
    tc = path == "tcgen05_tf32"
    rec = (path, bool(tc or (a_pre and tf32_on())), bool(tc or (b_pre and tf32_on() and not b_is_weight)))
    k = (kind,) + tuple(key)
    prev = CONV_TRACE.setdefault(k, rec)
    if prev != rec:
      # the same shape ran with differently prepared operands (e.g. an exact-fp32 filter gradient whose dy was stored
      # TF32-rounded for one layer and not for another): keep the union — the emulating oracle is a yard-stick for what
      # TF32 evaluation loses, the per-call truth goes to CONV_CHECK
      CONV_TRACE[k] = (prev[0] if prev[0] == rec[0] else "tcgen05_tf32", prev[1] or rec[1], prev[2] or rec[2])


def _fusable_relu(x):
  """(ref, leak) when the gradient w.r.t. `x` can take the (leaky-)ReLU mask of x's producer in the epilogue of the
  contraction that computes it: x is a ReLU output and this contraction is its only consumer in the running backward."""
  r = getattr(x, "relu_of", None)
  return r if (r is not None and _sole_consumer(x)) else None


def _premasked(g, y_id):
  return getattr(g, "premasked_for", None) == y_id


def _desc_key(d):
  up = 2 if d.upsample else 1
  return (d.n, d.h * up, d.w * up, d.cin, d.cout, d.kh, d.kw, d.stride)


_TC_NODES = ("conv2d", "conv2d_dgrad", "attention")
_PASS_NODES = ("avgpool2", "reshape")


def _grad_feeds_tc(t):
  """Will the gradient w.r.t. `t` be the dy operand of a tensor-core contraction?  (Then its producer stores it
  TF32-rounded and the contraction skips its rounding pass; a wrong guess only costs that pass.)"""
  if not tf32_on() or (t is not None and len(t.shape) == 4 and t.shape[-1] <= 4):
    return False          # (3-channel image-side contractions round their thin operand while gathering the patch tensor)
  for _ in range(4):
    if t is None or t.node is None:
      return False
    if t.node.name in _TC_NODES:
      return True
    if t.node.name not in _PASS_NODES:
      return False
    t = t.node.inputs[0]
  return False

ACT_RELU, ACT_LRELU, ACT_SIGMOID, ACT_TANH01 = 1, 2, 3, 4
LOSSES = {"non_saturating": 0, "hinge": 1, "wasserstein": 2, "least_squares": 3}


def init(device=0):
  """Bind this process to one GPU (one process per GPU) and load the C-ABI library."""
  if not torch.cuda.is_available():
    raise _lib.CganError("compare_gan_b200 needs a CUDA device: the product path has no CPU fallback")
  torch.cuda.set_device(device)
  _RT["lib"] = _lib.get_lib(device)
  _RT["device"] = torch.device("cuda", device)
  sync_stream()
  return _RT["lib"]


def lib():
  if _RT["lib"] is None:
    init(torch.cuda.current_device() if torch.cuda.is_available() else 0)
  return _RT["lib"]


def sync_stream():
  """Point the library at torch's current stream (call after switching streams / entering capture)."""
  _RT["lib"].set_stream(torch.cuda.current_stream().cuda_stream)


def empty(*shape):
  return DT(torch.empty(shape, dtype=torch.float32, device=_RT["device"]))


def from_numpy(a, req=False):
  import numpy as np
  a = np.asarray(a)
  t = torch.from_numpy(np.ascontiguousarray(a).reshape(a.shape)).to(_RT["device"])
  return DT(t.contiguous(), req)


def _call(name, *args):
  _RT["lib"].call(name, *args)


# ------------------------------------------------------------------------------------ basic helpers

def _grad_out(leaf, *shape):
  """Where the gradient w.r.t. `leaf` goes: the destination tape.backward's caller offered for it (its slot in the flat
  gradient buffer — no copy afterwards), else fresh memory."""
  s = _take_sink(leaf)
  if s is not None:
    n = 1
    for v in shape:
      n *= v
    if s.numel == n:
      return s.view(*shape)
  return empty(*shape)


def fill_(x, value):
  _call("fill", x.ptr, float(value), x.numel)
  return x


def zeros(*shape):
  return fill_(empty(*shape), 0.0)


def copy_(dst, src):
  assert dst.numel == src.numel
  _call("copy", dst.ptr, src.ptr, dst.numel)
  return dst


def reshape(x, *shape):
  """tf.reshape: zero-copy view, taped."""
  y = DT(x.t.view(*shape))
  y.tf32 = x.tf32
  xs = x.shape
  return attach("reshape", y, [x], lambda g, needs: [reshape(g, *xs)])


def add(a, b, round_tf32=False):
  assert a.shape == b.shape, (a.shape, b.shape)
  y = empty(*a.shape)
  rnd = bool(round_tf32) and tf32_on()
  _call("add_tf32", y.ptr, a.ptr, b.ptr, y.numel, int(rnd))
  y.tf32 = rnd
  return attach("add", y, [a, b], lambda g, needs: [g if needs[0] else None, g if needs[1] else None])


@_grad_accumulator
def add_grad(prev, g, tensor):
  """Gradient accumulation for tape.backward: the sum is stored TF32-rounded when it is about to feed tensor-core
  gradient contractions (the tensor it belongs to was produced by a convolution)."""
  return add(prev, g, round_tf32=_grad_feeds_tc(tensor))


def affine(x, a, c=0.0):
  """y = a*x + c  (sndcgan.py:108 `x*2-1`; loss weights)."""
  y = empty(*x.shape)
  _call("axpby", y.ptr, float(a), x.ptr, 0.0, None, float(c), y.numel)
  return attach("affine", y, [x], lambda g, needs: [affine(g, a)])


def axpy_(y, a, x):
  """y += a*x in place (gradient accumulation into flat buffers; untaped)."""
  _call("axpby", y.ptr, float(a), x.ptr, 1.0, y.ptr, 0.0, y.numel)
  return y


def concat_rows(a, b):
  """tf.concat([a, b], axis=0) (modular_gan.py:657)."""
  assert a.shape[1:] == b.shape[1:]
  y = empty(a.shape[0] + b.shape[0], *a.shape[1:])
  na = a.numel
  _call("copy", y.ptr, a.ptr, na)
  _call("copy", y.ptr + 4 * na, b.ptr, b.numel)
  ra = a.shape[0]

  def vjp(g, needs):
    return [slice_rows(g, 0, ra) if needs[0] else None, slice_rows(g, ra, g.shape[0]) if needs[1] else None]
  return attach("concat_rows", y, [a, b], vjp)


def slice_rows(x, lo, hi):
  """x[lo:hi] as a zero-copy view (tf.split on axis 0, modular_gan.py:660-661)."""
  y = DT(x.t[lo:hi])
  y.tf32 = x.tf32
  n0 = x.shape[0]

  def vjp(g, needs):
    full = zeros(*((n0,) + g.shape[1:]))
    per = g.numel // max(1, g.shape[0])
    _call("copy", full.ptr + 4 * lo * per, g.ptr, g.numel)
    return [full]
  return attach("slice_rows", y, [x], vjp)


def rot90(x, k):
  """Images rotated by k * 90 degrees (gans/utils.py:38-49, rotate_images); k in 1..3, square NHWC."""
  n, h, w, c = x.shape
  if h != w:
    raise ValueError("rot90 needs square images, got %dx%d" % (h, w))
  k = int(k) % 4
  if k == 0:
    return x
  y = empty(n, h, w, c)
  _call("rot90", y.ptr, x.ptr, n, h, c, k)
  return attach("rot90", y, [x], lambda g, needs: [rot90(g, 4 - k)])       # a permutation: the adjoint is the inverse


def rotation_loss(logits, num_rotations=4):
  """-mean log(softmax(logits)[r // m] + 1e-10) over the 4*m rows (gans/ssgan.py:205-213); a one-element device tensor."""
  rows, nrot = logits.shape
  if nrot != num_rotations or rows % nrot:
    raise ValueError("rotation_loss: logits must be [num_rotations * m, num_rotations], got %s" % (logits.shape,))
  loss, dl = empty(1), empty(rows, nrot)
  _call("rotation_loss", loss.ptr, dl.ptr, logits.ptr, rows, nrot)
  return attach("rotation_loss", loss, [logits], lambda g, needs: [_scale_by(dl, g)])


def row_has_label(y):
  """[N, 1] indicator: 1 where the (one-hot or soft) label row sums to more than 0.5, i.e. a label was passed
  (gans/s3gan.py:121-122).  A constant for differentiation."""
  rows, cols = y.shape
  out = empty(rows, 1)
  _call("row_has_label", out.ptr, y.ptr, rows, cols)
  return out


def argmax_one_hot(logits):
  """tf.one_hot(tf.arg_max(logits, 1), classes) (gans/s3gan.py:149-150); a constant for differentiation."""
  rows, cols = logits.shape
  out = empty(rows, cols)
  _call("argmax_one_hot", out.ptr, logits.ptr, rows, cols)
  return out


def softmax_xent(logits, labels, weights=None):
  """tf.losses.softmax_cross_entropy(labels, logits, weights=weights) (SUM_BY_NONZERO_WEIGHTS; gans/s3gan.py:312-313): a
  one-element device tensor, differentiable w.r.t. the logits."""
  rows, cols = logits.shape
  if labels.shape != (rows, cols) or (weights is not None and weights.numel != rows):
    raise ValueError("softmax_xent: labels %s / weights do not match logits %s" % (labels.shape, logits.shape))
  loss, dl = empty(1), empty(rows, cols)
  _call("softmax_xent", loss.ptr, dl.ptr, logits.ptr, labels.ptr, None if weights is None else weights.ptr, rows, cols)
  return attach("softmax_xent", loss, [logits], lambda g, needs: [_scale_by(dl, g)])


def concat_cols(a, b):
  """tf.concat([a, b], axis=1) for rank-2 tensors (resnet_biggan.py:254)."""
  n, ca, cb = a.shape[0], a.shape[1], b.shape[1]
  y = empty(n, ca + cb)
  _call("copy2d", y.ptr, ca + cb, 0, a.ptr, ca, 0, n, ca)
  _call("copy2d", y.ptr, ca + cb, ca, b.ptr, cb, 0, n, cb)

  def vjp(g, needs):
    return [slice_cols(g, 0, ca) if needs[0] else None, slice_cols(g, ca, ca + cb) if needs[1] else None]
  return attach("concat_cols", y, [a, b], vjp)


def slice_cols(x, lo, hi):
  """x[:, lo:hi] (tf.split on axis 1, resnet_biggan.py:251-252)."""
  n, c = x.shape
  y = empty(n, hi - lo)
  _call("copy2d", y.ptr, hi - lo, 0, x.ptr, c, lo, n, hi - lo)

  def vjp(g, needs):
    full = zeros(n, c)
    _call("copy2d", full.ptr, c, lo, g.ptr, hi - lo, 0, n, hi - lo)
    return [full]
  return attach("slice_cols", y, [x], vjp)


# ------------------------------------------------------------------------------------ contractions

def same_pad(n, k, s):
  """TF SAME: out=ceil(n/s), pad_before = max((out-1)*s+k-n, 0)//2."""
  out = -(-n // s)
  total = max((out - 1) * s + k - n, 0)
  return out, total // 2


def conv_desc(n, h, w, cin, cout, kh, kw, stride, upsample, padding="SAME"):
  vh, vw = (2 * h, 2 * w) if upsample else (h, w)
  if padding == "SAME":
    oh, pt = same_pad(vh, kh, stride)
    ow, pl = same_pad(vw, kw, stride)
  elif padding == "VALID":
    oh, pt = (vh - kh) // stride + 1, 0
    ow, pl = (vw - kw) // stride + 1, 0
  else:
    raise ValueError("padding must be SAME or VALID")
  return _lib.ConvDesc(n, h, w, cin, cout, kh, kw, stride, 1 if upsample else 0, oh, ow, pt, pl)


def _epilogue(bias=None, residual=None, mask=None, mask_leak=0.0, relu=False, round_out=False, in_tf32=False, ldy=0):
  flags = (_lib.CONV_RELU if relu else 0) | (_lib.CONV_ROUND_OUT if round_out else 0) | (_lib.CONV_IN_TF32 if in_tf32 else 0)
  return _lib.ConvEpilogue(None if bias is None else bias.ptr, None if residual is None else residual.ptr,
                           None if mask is None else mask.ptr, float(mask_leak), flags, int(ldy))


def _conv_fwd_raw(d, x, w, bias, relu=False, residual=None, round_out=False):
  y = empty(d.n, d.oh, d.ow, d.cout)
  rnd = bool(round_out) and tf32_on()
  ep = _epilogue(bias, residual, relu=relu, round_out=rnd, in_tf32=x.tf32 and tf32_on())
  _call("conv2d_fwd_ex", ctypes.byref(d), x.ptr, w.ptr, ctypes.byref(ep), y.ptr)
  _trace("fwd", _desc_key(d), x.tf32)
  y.tf32 = rnd
  if CONV_CHECK is not None:
    CONV_CHECK("fwd", d=d, x=x, w=w, bias=bias, residual=residual, relu=relu, round_out=rnd, out=y, arith=_arith(x.tf32))
  return y


def conv2d_relu(x, w, bias, stride=1, padding="SAME", sink=None, sink_off=0):
  """relu(conv2d(x, w) + bias) in one kernel; inference only (no tape).  With `sink` (a ChannelSink) the result is
  stored straight into channels [sink_off, sink_off + cout) of the wider NHWC tensor (tf.concat(axis=3) without the
  copy) and None is returned."""
  n, h, ww, cin = x.shape
  kh, kw, _, cout = w.shape
  d = conv_desc(n, h, ww, cin, cout, kh, kw, stride, False, padding)
  b = None if bias is None else bias.ptr
  if sink is not None:
    buf = sink.buffer(d.n, d.oh, d.ow)
    _call("conv2d_fwd_act_ld", ctypes.byref(d), x.ptr, w.ptr, b, ACT_RELU, buf.ptr + 4 * sink_off, sink.channels)
    return None
  y = empty(d.n, d.oh, d.ow, d.cout)
  _call("conv2d_fwd_act", ctypes.byref(d), x.ptr, w.ptr, b, ACT_RELU, y.ptr)
  return y


class ChannelSink(object):
  """The output of a channel concatenation, allocated when the first producer knows the spatial size."""

  def __init__(self, channels):
    self.channels, self.buf = channels, None

  def buffer(self, n, h, w):
    if self.buf is None:
      self.buf = empty(n, h, w, self.channels)
    elif self.buf.shape[:3] != (n, h, w):
      raise ValueError("concat: branch output %s does not match %s" % ((n, h, w), self.buf.shape[:3]))
    return self.buf

  def put(self, t, off):
    """Copies an already materialised branch (the pooling branches) into its slice."""
    n, h, w, c = t.shape
    buf = self.buffer(n, h, w)
    _call("copy2d", buf.ptr, self.channels, off, t.ptr, c, 0, n * h * w, c)


def conv2d(x, w, bias=None, stride=1, upsample=False, padding="SAME", relu=False, residual=None, round_out=False):
  """tf.nn.conv2d(..., "SAME") + bias (arch_ops.py:568-572); `upsample` fuses resnet_ops.unpool
  (resnet_ops.py:35-56, 122-123) without materialising the zeros.  w is HWIO.

  Epilogue fusions (include/cgan_b200.h, cgan_conv2d_fwd_ex): `residual` (same shape as the output) is added before the
  activation (the `h + shortcut` of resnet_ops.py:181), `relu` applies tf.nn.relu to the result (the pre-activation of
  the NEXT convolution, resnet_ops.py:174), `round_out` stores TF32-rounded values in math_mode 1 (the output only feeds
  tensor-core contractions)."""
  n, h, ww, cin = x.shape
  kh, kw, wcin, cout = w.shape
  if wcin != cin:
    raise ValueError("conv2d: kernel expects %d input channels, got %d" % (wcin, cin))
  d = conv_desc(n, h, ww, cin, cout, kh, kw, stride, upsample, padding)
  if residual is not None and residual.shape != (d.n, d.oh, d.ow, d.cout):
    raise ValueError("conv2d: residual shape %s does not match the output %s" % (residual.shape, (d.n, d.oh, d.ow, d.cout)))
  y = _conv_fwd_raw(d, x, w, bias, relu, residual, round_out)
  if relu and RELU_OBSERVERS:
    for fn in RELU_OBSERVERS:
      fn(y.t > 0)
  yv = DT(y.t) if relu else None        # y > 0  <=>  pre-activation > 0
  if relu:
    y.relu_of = (yv, 0.0)
  y_id = id(y)

  def vjp(g, needs):
    if relu and not _premasked(g, y_id):
      g = act_bwd(g, yv, ACT_RELU, round_tf32=True)
    return [conv2d_dgrad(d, g, w, round_out=_grad_feeds_tc(x), relu_mask=_fusable_relu(x), mask_for=x) if needs[0] else None,
            conv2d_wgrad(d, x, g, leaf=w) if needs[1] else None,
            colsum(reshape(g, -1, cout), leaf=bias) if (bias is not None and needs[2]) else None,
            g if (residual is not None and needs[3]) else None]
  return attach("conv2d", y, [x, w, bias, residual], vjp)


def conv2d_dgrad(d, dy, w, bias=None, round_out=False, relu_mask=None, mask_for=None):
  """Input gradient of conv2d == tf.nn.conv2d_transpose (+ bias, arch_ops.py:588-592).  `relu_mask` = (ref, leak): the
  result is the gradient w.r.t. a (leaky-)ReLU output `mask_for`; that ReLU's backward (g * [ref > 0 ? 1 : leak]) is applied
  in this kernel's epilogue and the result is tagged so the ReLU's own vjp passes it through."""
  dx = empty(d.n, d.h, d.w, d.cin)
  rnd = bool(round_out) and tf32_on()
  mref, mleak = relu_mask if relu_mask is not None else (None, 0.0)
  ep = _epilogue(bias, mask=mref, mask_leak=mleak, round_out=rnd, in_tf32=dy.tf32 and tf32_on())
  _call("conv2d_dgrad_ex", ctypes.byref(d), dy.ptr, w.ptr, ctypes.byref(ep), dx.ptr)
  _trace("dgrad", _desc_key(d), dy.tf32)
  dx.tf32 = rnd
  if mref is not None:
    dx.premasked_for = id(mask_for)
  if CONV_CHECK is not None:
    CONV_CHECK("dgrad", d=d, dy=dy, w=w, bias=bias, round_out=rnd, mask=mref, mask_leak=mleak, out=dx, arith=_arith(dy.tf32))
  cin = d.cin

  def vjp(g, needs):   # linear in dy and in w
    return [_taped_fwd(d, g, w, round_out=_grad_feeds_tc(dy)) if needs[0] else None,
            conv2d_wgrad(d, g, dy, leaf=w) if needs[1] else None,
            colsum(reshape(g, -1, cin), leaf=bias) if (bias is not None and needs[2]) else None]
  return attach("conv2d_dgrad", dx, [dy, w, bias], vjp)


def _taped_fwd(d, x, w, round_out=False):
  y = _conv_fwd_raw(d, x, w, None, round_out=round_out)

  def vjp(g, needs):
    return [conv2d_dgrad(d, g, w, round_out=_grad_feeds_tc(x), relu_mask=_fusable_relu(x), mask_for=x) if needs[0] else None,
            conv2d_wgrad(d, x, g, leaf=w) if needs[1] else None]
  return attach("conv2d", y, [x, w], vjp)


def conv2d_wgrad(d, x, dy, leaf=None):
  """Filter gradient (TF Conv2DBackpropFilter); deterministic split-K.  `leaf`: the kernel variable, see _grad_out."""
  dw = _grad_out(leaf, d.kh, d.kw, d.cin, d.cout)
  flags = 0
  if tf32_on():
    flags = (_lib.CONV_IN_TF32 if x.tf32 else 0) | (_lib.CONV_IN2_TF32 if dy.tf32 else 0)
  _call("conv2d_wgrad_ex", ctypes.byref(d), x.ptr, dy.ptr, flags, dw.ptr)
  _trace("wgrad", _desc_key(d), x.tf32, dy.tf32, b_is_weight=False)
  if CONV_CHECK is not None:
    CONV_CHECK("wgrad", d=d, x=x, dy=dy, out=dw, arith=_arith(x.tf32, dy.tf32, b_is_weight=False))

  def vjp(g, needs):
    raise NotImplementedError("third-order differentiation through conv2d_wgrad is not needed on this path")
  return attach("conv2d_wgrad", dw, [x, dy], vjp)


def deconv2d(x, w, bias, out_hw, stride):
  """tf.nn.conv2d_transpose + bias (arch_ops.py:579-592).  w is [kh,kw,cout,cin(=x channels)]: as an HWIO conv
  kernel it maps the deconv OUTPUT (cout channels) to x, so deconv(x) is that conv's input gradient; the bias is added
  in the same kernel's epilogue."""
  n, h, ww, cin = x.shape
  kh, kw, cout, wcin = w.shape
  if wcin != cin:
    raise ValueError("deconv2d: kernel expects %d input channels, got %d" % (wcin, cin))
  oh, ow = out_hw
  d = conv_desc(n, oh, ow, cout, cin, kh, kw, stride, False)
  if (d.oh, d.ow) != (h, ww):
    raise ValueError("deconv2d: output shape %s incompatible with input %s" % ((oh, ow), (h, ww)))
  return conv2d_dgrad(d, x, w, bias)


def matmul(a, b, ta=False, tb=False, leaf=None):
  """tf.matmul (arch_ops.py:548).  `leaf`: the variable this product is the gradient of, see _grad_out."""
  m = a.shape[1] if ta else a.shape[0]
  k = a.shape[0] if ta else a.shape[1]
  kb = b.shape[1] if tb else b.shape[0]
  n = b.shape[0] if tb else b.shape[1]
  if k != kb:
    raise ValueError("matmul: inner dimensions differ: %d vs %d" % (k, kb))
  c = _grad_out(leaf, m, n)
  _call("gemm", int(ta), int(tb), m, n, k, 1.0, a.ptr, a.shape[1], b.ptr, b.shape[1], 0.0, c.ptr, n)

  def vjp(g, needs):
    ga = gb = None
    if needs[0]:
      ga = matmul(b, g, tb, True) if ta else matmul(g, b, False, not tb)
    if needs[1]:
      gb = matmul(g, a, True, ta, leaf=b) if tb else matmul(a, g, not ta, False, leaf=b)
    return [ga, gb]
  return attach("matmul", c, [a, b], vjp)


def bmm(a, b, ta=False, tb=False):
  """Batched tf.matmul on rank-3 tensors (arch_ops.py:744, 753)."""
  bsz = a.shape[0]
  m = a.shape[2] if ta else a.shape[1]
  k = a.shape[1] if ta else a.shape[2]
  n = b.shape[1] if tb else b.shape[2]
  c = empty(bsz, m, n)
  _call("gemm_batched", int(ta), int(tb), m, n, k, 1.0, a.ptr, a.shape[2], a.shape[1] * a.shape[2],
        b.ptr, b.shape[2], b.shape[1] * b.shape[2], 0.0, c.ptr, n, m * n, bsz)
  _trace("bmm", (bsz, int(ta), int(tb), m, n, k))
  if CONV_CHECK is not None:
    CONV_CHECK("bmm", a=a, b=b, ta=ta, tb=tb, out=c, arith=_arith())

  def vjp(g, needs):
    ga = gb = None
    if needs[0]:
      ga = bmm(b, g, tb, True) if ta else bmm(g, b, False, not tb)
    if needs[1]:
      gb = bmm(g, a, True, ta) if tb else bmm(a, g, not ta, False)
    return [ga, gb]
  return attach("bmm", c, [a, b], vjp)


def round_tf32(x):
  """x rounded to the nearest TF32 value (identity for the gradient, like the rounding a tensor-core contraction applies to
  its operands); a no-op when the producer already stored x rounded."""
  if x.tf32 or not tf32_on():
    return x
  y = empty(*x.shape)
  _call("round_tf32", y.ptr, x.ptr, y.numel)
  y.tf32 = True
  return attach("round_tf32", y, [x], lambda g, needs: [g])


def attention_shape_ok(bsz, lq, lk, dk, dv):
  """Do the fused wgmma attention kernels take this shape in the current math mode?"""
  return bool(tf32_on() and lib().attention_supported(bsz, lq, lk, dk, dv))


def attention_fused_ok(theta, phi, g):
  bsz, lq, dk = theta.shape
  return attention_shape_ok(bsz, lq, phi.shape[1], dk, g.shape[2])


def attention(theta, phi, g):
  """softmax(theta phi^T) g per image — tf.matmul(theta, phi, transpose_b=True) -> tf.nn.softmax -> tf.matmul(attn, g)
  (arch_ops.py:744-753).  In math_mode 1, for shapes the fused wgmma kernels take (csrc/attn_tc.cu: BigGAN's 4096 x 1024
  scores at 24 / 12 key channels), ONE kernel per direction keeps the scores in registers; otherwise the three
  ops are composed as the reference writes them."""
  if not attention_fused_ok(theta, phi, g):
    return bmm(softmax(bmm(theta, phi, False, True)), g)
  bsz, lq, dk = theta.shape
  lk, dv = g.shape[1], g.shape[2]
  q, k, v = round_tf32(theta), round_tf32(phi), round_tf32(g)
  out = empty(bsz, lq, dv)
  lse = empty(bsz, lq)
  _call("attention_fwd", q.ptr, k.ptr, v.ptr, out.ptr, lse.ptr, bsz, lq, lk, dk, dv)
  _trace("attention", (bsz, lq, lk, dk, dv), True, True, b_is_weight=False)
  if CONV_CHECK is not None:
    CONV_CHECK("attention", q=q, k=k, v=v, out=out, lse=lse)
  ov = DT(out.t)

  def vjp(gout, needs):
    _no_second_order("attention")
    go = gout
    if not go.tf32:
      go = empty(*gout.shape)
      _call("round_tf32", go.ptr, gout.ptr, go.numel)
    dq, dkk, dvv = empty(bsz, lq, dk), empty(bsz, lk, dk), empty(bsz, lk, dv)
    _call("attention_bwd", q.ptr, k.ptr, v.ptr, ov.ptr, lse.ptr, go.ptr, dq.ptr, dkk.ptr, dvv.ptr, bsz, lq, lk, dk, dv)
    if CONV_CHECK is not None:
      CONV_CHECK("attention_bwd", q=q, k=k, v=v, out=ov, lse=lse, dout=go, dq=dq, dk=dkk, dv=dvv)
    return [dq, dkk, dvv]
  return attach("attention", out, [q, k, v], vjp)


def colsum(x2, groups=1, leaf=None):
  """Per-channel sum over rows (bias / beta gradients).  `leaf`: the variable this is the gradient of, see _grad_out."""
  rows, c = x2.shape
  out = _grad_out(leaf, c) if groups == 1 else empty(groups, c)
  _call("colsum", out.ptr, x2.ptr, groups, rows // groups, c)
  return out   # leaf of the backward pass: never differentiated again


def bias_add(x, bias):
  c = x.shape[-1]
  y = empty(*x.shape)
  _call("bias_add", y.ptr, x.ptr, bias.ptr, x.numel // c, c)

  def vjp(g, needs):
    return [g if needs[0] else None, colsum(reshape(g, -1, c), leaf=bias) if needs[1] else None]
  return attach("bias_add", y, [x, bias], vjp)


# ------------------------------------------------------------------------------------ pointwise / pooling

RELU_OBSERVERS = []     # test hook: callables receiving the boolean "input > 0" mask of every (leaky-)ReLU evaluated


def act(x, kind, leak=0.0, round_tf32=False):
  """Pointwise activation; `round_tf32` (math_mode 1): the result only feeds tensor-core contractions, store it
  TF32-rounded so that they skip their operand-rounding pass."""
  if RELU_OBSERVERS and kind in (ACT_RELU, ACT_LRELU):
    for fn in RELU_OBSERVERS:
      fn(x.t > 0)
  y = empty(*x.shape)
  rnd = bool(round_tf32) and tf32_on()
  _call("act_fwd", y.ptr, x.ptr, kind | (_lib.ACT_ROUND_TF32 if rnd else 0), float(leak), y.numel)
  y.tf32 = rnd or (kind == ACT_RELU and x.tf32)
  # a closure must never hold its own output DT (that would be a DT -> node -> closure -> DT reference cycle and delay
  # freeing the stash until a cyclic GC pass): wrap the storage in a fresh, tape-less DT instead
  ref = x if kind in (ACT_RELU, ACT_LRELU) else DT(y.t)
  if kind in (ACT_RELU, ACT_LRELU):
    y.relu_of = (DT(x.t), float(leak) if kind == ACT_LRELU else 0.0)
  y_id = id(y)

  def vjp(g, needs):
    if _premasked(g, y_id):
      return [g]                      # the producing contraction applied this activation's mask in its epilogue
    return [act_bwd(g, ref, kind, leak, round_tf32=_grad_feeds_tc(x))]
  return attach("act%d" % kind, y, [x], vjp)


def act_bwd(g, ref, kind, leak=0.0, round_tf32=False):
  dx = empty(*g.shape)
  rnd = bool(round_tf32) and tf32_on()
  _call("act_bwd", dx.ptr, g.ptr, ref.ptr, kind | (_lib.ACT_ROUND_TF32 if rnd else 0), float(leak), dx.numel)
  dx.tf32 = rnd or (kind == ACT_RELU and g.tf32)        # a 0/1 mask keeps TF32 values TF32

  def vjp(gg, needs):
    if kind not in (ACT_RELU, ACT_LRELU):
      raise NotImplementedError("second derivative only needed for piecewise-linear activations")
    return [act_bwd(gg, ref, kind, leak, round_tf32=_grad_feeds_tc(g))]   # the mask is constant almost everywhere
  return attach("act_bwd%d" % kind, dx, [g], vjp)


def relu(x, round_tf32=False):
  return act(x, ACT_RELU, round_tf32=round_tf32)


def lrelu(x, leak=0.2, round_tf32=False):
  return act(x, ACT_LRELU, leak, round_tf32=round_tf32)


def sigmoid(x):
  return act(x, ACT_SIGMOID)


def tanh01(x):
  """(tanh(x)+1)/2 (sndcgan.py:74-78, resnet_biggan.py:301)."""
  return act(x, ACT_TANH01)


def avgpool2(x):
  """tf.nn.pool AVG 2x2 s2 (resnet_ops.py:131-133)."""
  n, h, w, c = x.shape
  y = empty(n, h // 2, w // 2, c)
  _call("avgpool2_fwd", y.ptr, x.ptr, n, h, w, c)
  return attach("avgpool2", y, [x], lambda g, needs: [avgpool2_bwd(g, h, w)])


def avgpool2_bwd(g, h, w):
  n, _, _, c = g.shape
  dx = empty(n, h, w, c)
  _call("avgpool2_bwd", dx.ptr, g.ptr, n, h, w, c)
  dx.tf32 = g.tf32          # g / 4 is exact
  return attach("avgpool2_bwd", dx, [g], lambda gg, needs: [avgpool2(gg)])


_UNPOOL_MASKS = {}


def unpool(x):
  """resnet_ops.unpool materialised (resnet_ops.py:35-56): zero insertion to twice the size, x at the even positions.
  Only the identity shortcut of resnet_biggan_deep's up blocks needs the tensor itself (convolutions over an unpooled
  input use conv2d(upsample=True) and never build it).  Composed of two existing kernels: avgpool2's adjoint spreads
  x / 4 over each 2x2 cell, a per-pixel scale (4 at the even-even pixel, 0 elsewhere) keeps the corner — exact in fp32,
  and differentiable to any order because both parts are taped ops."""
  import numpy as np
  n, h, w, c = x.shape
  key = (n, h, w, str(_RT["device"]))
  if key not in _UNPOOL_MASKS:          # built once per shape, i.e. during the eager warm-up that precedes graph capture
    cell = np.zeros((2 * h, 2 * w), np.float32)
    cell[::2, ::2] = 4.0
    _UNPOOL_MASKS[key] = from_numpy(np.tile(cell.reshape(1, -1), (n, 1)).reshape(-1))
  spread = avgpool2_bwd(x, 2 * h, 2 * w)
  return reshape(rowscale(reshape(spread, -1, c), _UNPOOL_MASKS[key]), n, 2 * h, 2 * w, c)


def maxpool2(x):
  """tf.layers.max_pooling2d(2, 2) (arch_ops.py:741, 750)."""
  n, h, w, c = x.shape
  y = empty(n, h // 2, w // 2, c)
  _call("maxpool2_fwd", y.ptr, x.ptr, n, h, w, c)
  y.tf32 = x.tf32           # a maximum of TF32 values is one of them

  def vjp(g, needs):
    _no_second_order("maxpool2")
    dx = empty(n, h, w, c)
    _call("maxpool2_bwd", dx.ptr, g.ptr, x.ptr, n, h, w, c)
    return [dx]
  return attach("maxpool2", y, [x], vjp)


def pool2d(x, k, stride, padding, mode):
  """tf.nn.max_pool / tf.nn.avg_pool (TF-GAN's Inception graph); inference only."""
  n, h, w, c = x.shape
  if padding == "SAME":
    oh, pt = same_pad(h, k, stride)
    ow, pl = same_pad(w, k, stride)
  else:
    oh, pt, ow, pl = (h - k) // stride + 1, 0, (w - k) // stride + 1, 0
  y = empty(n, oh, ow, c)
  _call("pool2d_fwd", y.ptr, x.ptr, n, h, w, c, k, stride, pt, pl, oh, ow, 0 if mode == "max" else 1)
  return y


def concat_channels(xs):
  """tf.concat(axis=3) of NHWC tensors (Inception mixed blocks); inference only."""
  n, h, w = xs[0].shape[:3]
  ctot = sum(t.shape[3] for t in xs)
  y = empty(n, h, w, ctot)
  off = 0
  for t in xs:
    c = t.shape[3]
    _call("copy2d", y.ptr, ctot, off, t.ptr, c, 0, n * h * w, c)
    off += c
  return y


def resize_bilinear(x, oh, ow, inception_scale=False):
  """tf.image.resize_bilinear (align_corners=False); with inception_scale also (v*255-128)/128 (eval_utils.py:157-175)."""
  n, h, w, c = x.shape
  y = empty(n, oh, ow, c)
  _call("resize_bilinear", y.ptr, x.ptr, n, h, w, c, oh, ow, 1 if inception_scale else 0)
  return y


def ssim_terms(images, pairs, levels, filter_size, filter_width, max_val):
  """Per-scale SSIM terms of image pairs of one set (metrics/image_similarity.py:85-211, 239-333): images [n,h,w,c] DT
  with values in [0, max_val], pairs int [npairs, 2] (host) indices into it.  Returns numpy [npairs, levels, c] float32:
  the pixel mean of cs at levels 0..levels-2 and of luminance*cs at the last level, before the relu."""
  import numpy as np
  n, h, w, c = images.shape
  pr = np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))
  out = empty(pr.shape[0], int(levels), c)
  _call("ssim_terms", out.ptr, images.ptr, n, h, w, c, pr.ctypes.data, pr.shape[0], int(levels), int(filter_size),
        float(filter_width), float(max_val))
  return out.cpu()


def globalpool(x, mean):
  """tf.reduce_mean / reduce_sum over axes [1,2] (resnet_cifar.py:156, resnet_biggan.py:405)."""
  n, h, w, c = x.shape
  scale = 1.0 / (h * w) if mean else 1.0
  y = empty(n, c)
  _call("globalpool_fwd", y.ptr, x.ptr, n, h * w, c, scale)
  return attach("globalpool", y, [x], lambda g, needs: [globalpool_bwd(g, h, w, scale)])


def globalpool_bwd(g, h, w, scale):
  n, c = g.shape
  dx = empty(n, h, w, c)
  _call("globalpool_bwd", dx.ptr, g.ptr, n, h * w, c, scale)

  def vjp(gg, needs):
    y = empty(n, c)
    _call("globalpool_fwd", y.ptr, gg.ptr, n, h * w, c, scale)
    return [attach("globalpool", y, [gg], lambda g3, needs3: [globalpool_bwd(g3, h, w, scale)])]
  return attach("globalpool_bwd", dx, [g], vjp)


def softmax(x):
  """tf.nn.softmax over the last axis (arch_ops.py:745)."""
  cols = x.shape[-1]
  rows = x.numel // cols
  shape = x.shape
  y = empty(*shape)
  _call("softmax_fwd", y.ptr, x.ptr, rows, cols)
  yv = DT(y.t)

  def vjp(g, needs):
    _no_second_order("softmax")
    dx = empty(*shape)
    _call("softmax_bwd", dx.ptr, g.ptr, yv.ptr, rows, cols)
    return [dx]
  return attach("softmax", y, [x], vjp)


def rowdot(a, b):
  """sum(a*b, axis=1, keepdims=True) (resnet_biggan.py:423)."""
  rows, cols = a.shape
  y = empty(rows, 1)
  _call("rowdot", y.ptr, a.ptr, b.ptr, rows, cols)
  return attach("rowdot", y, [a, b],
                lambda g, needs: [rowscale(b, g) if needs[0] else None, rowscale(a, g) if needs[1] else None])


def rowscale(a, s):
  rows, cols = a.shape
  y = empty(rows, cols)
  _call("rowscale", y.ptr, a.ptr, s.ptr, rows, cols)
  return attach("rowscale", y, [a, s],
                lambda g, needs: [rowscale(g, s) if needs[0] else None, rowdot(g, a) if needs[1] else None])


def scale_by_param(x, s):
  """x * s with s a scalar parameter on device (non_local_block sigma, arch_ops.py:755-758)."""
  y = empty(*x.shape)
  _call("scale_by_dev", y.ptr, x.ptr, s.ptr, 1.0, 0, y.numel)

  def vjp(g, needs):
    _no_second_order("scale_by_param")
    gx = gs = None
    if needs[0]:
      gx = empty(*x.shape)
      _call("scale_by_dev", gx.ptr, g.ptr, s.ptr, 1.0, 0, gx.numel)
    if needs[1]:
      gs = empty(*s.shape)
      _call("dot", gs.ptr, g.ptr, x.ptr, x.numel)
    return [gx, gs]
  return attach("scale_by_param", y, [x, s], vjp)


def one_hot(labels_i32, classes):
  """tf.one_hot (modular_gan.py:359-363); labels: int32 device tensor wrapped in a DT."""
  n = labels_i32.t.shape[0]
  y = empty(n, classes)
  _call("one_hot", y.ptr, labels_i32.ptr, n, classes)
  return y


def interpolate(x, xf, alpha):
  """x + alpha*(x_fake - x), alpha [B,1,1,1] (penalty_lib.py:74-75).  Result is a fresh leaf."""
  y = empty(*x.shape)
  _call("interpolate", y.ptr, x.ptr, xf.ptr, alpha.ptr, x.shape[0], x.numel // x.shape[0])
  return y


# ------------------------------------------------------------------------------------ batch norm

class BNState(object):
  """Per-layer buffers: moving averages or accumulators (arch_ops.py:66-191) and scratch."""
  __slots__ = ("moving_mean", "moving_var", "accu_mean", "accu_var", "accu_counter", "update_accus")

  def __init__(self):
    self.moving_mean = self.moving_var = None
    self.accu_mean = self.accu_var = self.accu_counter = self.update_accus = None


def bn_train(x, gamma, beta, eps, state=None, decay=0.999, cond=False, relu_after=False, allreduce=None, world=1,
             round_out=False):
  """Training-mode standardize_batch (+ gamma/beta) (arch_ops.py:194-319, 353-366, 435-444).

  gamma/beta: [C] DTs, or [N,C] when cond (conditional BN); either may be None.
  allreduce(stats_dt) sums a [2C] buffer over replicas (cross-replica moments, tpu_ops.py:94-125).
  """
  c = x.shape[-1]
  rows = x.numel // c
  rps = rows // x.shape[0]
  stats = empty(2 * c)
  _call("bn_moments", stats.ptr, x.ptr, rows, c)
  if allreduce is not None and world > 1:
    allreduce(stats)
    _call("axpby", stats.ptr, 1.0 / world, stats.ptr, 0.0, None, 0.0, 2 * c)
  mv = empty(2 * c)
  mm = state.moving_mean if state is not None else None
  mvv = state.moving_var if state is not None else None
  _call("bn_finalize", mv.ptr, stats.ptr, c, None if mm is None else mm.ptr, None if mvv is None else mvv.ptr,
        float(decay))
  y = empty(*x.shape)
  rnd = bool(round_out) and tf32_on()
  _call("bn_apply", y.ptr, x.ptr, rows, c, rps, mv.ptr, float(eps), None if gamma is None else gamma.ptr,
        None if beta is None else beta.ptr, int(cond), (1 if relu_after else 0) | (_lib.ACT_ROUND_TF32 if rnd else 0))
  y.tf32 = rnd

  yv = DT(y.t) if relu_after else None
  if relu_after:
    y.relu_of = (yv, 0.0)
  y_id = id(y)
  if relu_after and RELU_OBSERVERS:
    for fn in RELU_OBSERVERS:
      fn(y.t > 0)

  def vjp(g, needs):
    _no_second_order("bn_train")
    if relu_after and not _premasked(g, y_id):
      g = act_bwd(g, yv, ACT_RELU)    # y>0 <=> pre-activation>0
    sums = empty(2 * c)
    dgamma = dbeta = None
    if gamma is not None and needs[1]:
      dgamma = _grad_out(gamma, *gamma.shape)
    if beta is not None and needs[2]:
      dbeta = _grad_out(beta, *beta.shape)
    with no_record():
      _call("bn_bwd_reduce", sums.ptr, None if dgamma is None else dgamma.ptr, None if dbeta is None else dbeta.ptr,
            g.ptr, x.ptr, rows, c, rps, mv.ptr, float(eps), None if gamma is None else gamma.ptr, int(cond))
      count = rows
      if allreduce is not None and world > 1:
        allreduce(sums)
        count = rows * world
      dx = None
      if needs[0]:
        dx = empty(*x.shape)
        rnd_dx = _grad_feeds_tc(x)
        _call("bn_bwd_apply", dx.ptr, g.ptr, x.ptr, rows, c, rps, mv.ptr, float(eps),
              None if gamma is None else gamma.ptr, int(cond), sums.ptr, 1.0 / count, int(rnd_dx))
        dx.tf32 = rnd_dx
    return [dx, dgamma, dbeta]
  return attach("bn_train", y, [x, gamma, beta], vjp)


def bn_infer(x, gamma, beta, eps, state, use_moving_averages, cond=False, relu_after=False, round_out=False):
  """Inference-mode standardize_batch: moving averages (arch_ops.py:66-119) or accumulators (:122-191)."""
  c = x.shape[-1]
  rows = x.numel // c
  rps = rows // x.shape[0]
  if use_moving_averages:
    mv = empty(2 * c)
    _call("copy", mv.ptr, state.moving_mean.ptr, c)
    _call("copy", mv.ptr + 4 * c, state.moving_var.ptr, c)
  else:
    stats = empty(2 * c)
    _call("bn_moments", stats.ptr, x.ptr, rows, c)
    batch = empty(2 * c)
    _call("bn_finalize", batch.ptr, stats.ptr, c, None, None, 0.0)
    mv = empty(2 * c)
    _call("bn_accumulate", mv.ptr, batch.ptr, c, state.accu_mean.ptr, state.accu_var.ptr, state.accu_counter.ptr,
          state.update_accus.ptr)
  y = empty(*x.shape)
  rnd = bool(round_out) and tf32_on()
  _call("bn_apply", y.ptr, x.ptr, rows, c, rps, mv.ptr, float(eps), None if gamma is None else gamma.ptr,
        None if beta is None else beta.ptr, int(cond), (1 if relu_after else 0) | (_lib.ACT_ROUND_TF32 if rnd else 0))
  y.tf32 = rnd
  return y


# ------------------------------------------------------------------------------------ spectral norm

def spectral_normalize(w, u, left, eps=1e-12):
  """arch_ops.py:453-535: one power iteration, `u` (persistent state) updated in place, returns w/sigma.  Inside a
  `sn_batch` scope the small weights of a network are served from ONE batched launch (see SNBatch)."""
  rows = w.numel // w.shape[-1]
  cols = w.shape[-1]
  batch = _SN_SCOPE[-1]
  if batch is not None:
    hit = batch.lookup(w, u, left, eps)
    if hit is not None:
      wbar, v, sigma, u_used = hit
      return _sn_attach(w, wbar, rows, cols, left, u_used, v, sigma)
  v = empty(cols if left else rows)
  sigma = empty(1)
  wbar = empty(*w.shape)
  _call("spectral_norm", w.ptr, rows, cols, int(left), float(eps), u.ptr, v.ptr, sigma.ptr, wbar.ptr)
  # the backward needs u AFTER this call's update; later calls overwrite u_var, so keep a copy
  u_used = empty(*u.shape)
  _call("copy", u_used.ptr, u.ptr, u.numel)
  return _sn_attach(w, wbar, rows, cols, left, u_used, v, sigma)


def _sn_attach(w, wbar, rows, cols, left, u_used, v, sigma):
  wbar_v = DT(wbar.t)

  def vjp(g, needs):
    _no_second_order("spectral_normalize")
    dw = _grad_out(w, *w.shape)
    _call("spectral_norm_bwd", dw.ptr, g.ptr, wbar_v.ptr, rows, cols, int(left), u_used.ptr, v.ptr, sigma.ptr)
    return [dw]
  return attach("spectral_norm", wbar, [w], vjp)


_SN_SCOPE = [None]
SN_BATCH_MAX_ELEMS = 1 << 18        # weights up to 1 MB go through the one-CTA-per-weight batched kernel
SN_BATCH_MAX_DIMS = 12288           # rows + cols (shared-memory vectors of that CTA)


class SNBatch(object):
  """The spectrally normalised weights of one network (generator or discriminator), learned on its first call.  From
  the second call on, entering the scope runs the power iteration of all SMALL weights (the 3x3x128x128 kernels of
  resnet_cifar's discriminator, SNDCGAN's first layers, the conditional-BN projections of BigGAN) in one launch of
  cgan_spectral_norm_batched, and `spectral_normalize` hands out views of its outputs — same arithmetic, same one
  iteration per call site and weight (arch_ops.py:503-531), ~7 launches per weight fewer.  Large weights keep the
  per-weight kernels, which stream them from HBM with the whole GPU."""

  def __init__(self):
    self.plan, self.keys, self.complete = [], set(), False
    self.table, self.table_ptrs, self.results = None, None, {}

  def lookup(self, w, u, left, eps):
    rows, cols = w.numel // w.shape[-1], w.shape[-1]
    if not self.complete:
      small = rows * cols <= SN_BATCH_MAX_ELEMS and rows + cols <= SN_BATCH_MAX_DIMS
      if small and id(w) not in self.keys and w.node is None:      # a raw variable (not e.g. an EMA-swapped temporary)
        self.keys.add(id(w))
        self.plan.append((w, u, bool(left), float(eps)))
      return None
    return self.results.pop(id(w), None)

  def run(self):
    """Launch the batched iteration for this call; fills self.results {id(w): (wbar, v, sigma, u_used)}."""
    import numpy as np
    self.results = {}
    if not self.plan:
      return
    eps = self.plan[0][3]
    ptrs = [(w.ptr, u.ptr) for w, u, _, _ in self.plan]
    if self.table is None or self.table_ptrs != ptrs:
      items = np.zeros(len(self.plan), dtype=[("w", "<u8"), ("u", "<u8"), ("rows", "<i4"), ("cols", "<i4"), ("left", "<i4"),
                                              ("reserved", "<i4"), ("wbar_off", "<i8"), ("v_off", "<i8"), ("u_off", "<i8")])
      wo = vo = uo = 0
      self.layout = []
      for i, (w, u, left, e) in enumerate(self.plan):
        rows, cols = w.numel // w.shape[-1], w.shape[-1]
        nu, nv = (rows, cols) if left else (cols, rows)
        items[i] = (w.ptr, u.ptr, rows, cols, int(left), 0, wo, vo, uo)
        self.layout.append((wo, vo, uo, rows, cols, nu, nv))
        wo += (rows * cols + 63) // 64 * 64
        vo += (nv + 63) // 64 * 64
        uo += (nu + 63) // 64 * 64
      self.sizes = (wo, vo, uo)
      self.max_dims = max(l[3] + l[4] for l in self.layout)
      self.table = torch.from_numpy(items.view(np.uint8).copy()).to(_RT["device"])
      self.table_ptrs = ptrs
    wo, vo, uo = self.sizes
    wbar_all, v_all, u_all, sig_all = empty(wo), empty(vo), empty(uo), empty(len(self.plan))
    _call("spectral_norm_batched", self.table.data_ptr(), len(self.plan), int(self.max_dims), float(eps), wbar_all.ptr,
          v_all.ptr, sig_all.ptr, u_all.ptr)
    for i, ((w, u, left, e), (wof, vof, uof, rows, cols, nu, nv)) in enumerate(zip(self.plan, self.layout)):
      self.results[id(w)] = (DT(wbar_all.t[wof:wof + rows * cols].view(w.shape)), DT(v_all.t[vof:vof + nv]),
                             DT(sig_all.t[i:i + 1]), DT(u_all.t[uof:uof + nu]))


class sn_batch(object):
  """`with sn_batch(state):` around one generator / discriminator call (architectures/abstract_arch.py)."""

  def __init__(self, state):
    self.state = state

  def __enter__(self):
    st = self.state
    if st.complete and all(e == st.plan[0][3] for _, _, _, e in st.plan):
      st.run()
    _SN_SCOPE.append(st)
    return st

  def __exit__(self, exc_type, *a):
    _SN_SCOPE.pop()
    st = self.state
    if exc_type is None and not st.complete:
      st.complete = True              # the first call has seen every spectrally normalised weight of the network
    leftover, st.results = st.results, {}
    if exc_type is None and leftover:
      raise RuntimeError("%d spectrally normalised weights were iterated by the batched launch but not used by this call: "
                         "their u vectors advanced without a call site" % len(leftover))


# ------------------------------------------------------------------------------------ losses / penalties

def _scale_by(x, g):
  """x * g[0] with g a one-element device tensor (chain rule through a scalar loss)."""
  y = empty(*x.shape)
  _call("scale_by_dev", y.ptr, x.ptr, g.ptr, 1.0, 0, y.numel)
  return y


def gan_losses(kind, d_real_logits, d_fake_logits):
  """gans/loss_lib.py:53-148 in one fused kernel.  Returns (d_loss, d_loss_real, d_loss_fake, g_loss) as
  one-element device tensors; d_loss and g_loss are differentiable wrt both logit tensors."""
  b = d_real_logits.shape[0]
  out4 = empty(4)
  dl_d = empty(2 * b, 1)
  dl_g = empty(2 * b, 1)
  _call("gan_loss", LOSSES[kind], d_real_logits.ptr, d_fake_logits.ptr, b, out4.ptr, dl_d.ptr, 0)
  _call("gan_loss", LOSSES[kind], d_real_logits.ptr, d_fake_logits.ptr, b, out4.ptr, dl_g.ptr, 1)

  def make(idx, dl):
    loss = DT(out4.t[idx:idx + 1])

    def vjp(g, needs):
      s = _scale_by(dl, g)
      return [DT(s.t[:b]) if needs[0] else None, DT(s.t[b:]) if needs[1] else None]
    return attach("gan_loss", loss, [d_real_logits, d_fake_logits], vjp)
  return make(0, dl_d), DT(out4.t[1:2]), DT(out4.t[2:3]), make(3, dl_g)


def gp_penalty(g):
  """gans/penalty_lib.py:78-81 on g = d logits / d x_hat: mean((sqrt(1e-4 + sum g^2) - 1)^2)."""
  n = g.shape[0]
  pen = empty(1)
  dg = empty(*g.shape)
  _call("gp_penalty", pen.ptr, dg.ptr, g.ptr, n, g.numel // n, 1.0)
  return attach("gp_penalty", pen, [g], lambda gg, needs: [_scale_by(dg, gg)])


def set_math_mode(mode):
  """0: exact fp32 SIMT contractions; 1: wgmma TF32 tensor-core convolutions where the shape allows
  (operands rounded to nearest TF32, fp32 accumulation)."""
  _call("ctx_set_math_mode", int(mode))
  _RT["math_mode"] = int(mode)
