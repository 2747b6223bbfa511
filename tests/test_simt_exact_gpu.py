"""The exact-fp32 kernels of math_mode 0 (the gather-GEMM of csrc/gemm.cu, the streaming image-side kernels of thin.cu, the
column reductions and the spectral-norm iterations of norm.cu), bit for bit and element by element against float64.

These kernels never round their operands.  With operands that are small integers, every product and every partial sum is
an integer below 2^24 and therefore exact in fp32, in ANY summation order:

    R = floor(sqrt((2^24 - 1) / (K + extra)))      (K terms of the contraction, `extra` for bias / residual / beta*C)

so the result must equal the float64 contraction cast to float32 exactly (np.testing.assert_array_equal semantics: the
two zeros are equal).  Epilogue steps that round once (alpha / beta scaling, ReLU, the (leaky-)ReLU mask gate, TF32 output
rounding) are reproduced in numpy float32.  Any missing, duplicated or misplaced term at any element fails, and is
reported as the first differing element decoded to (n, y, x, c), (kh, kw, ci, co) or (batch, row, col).

Every output lives inside a larger buffer whose margins (and the stride gaps of a padded leading dimension, a batch stride
or a channel slice) hold a NaN sentinel; their bits must survive the call, so a stray write fails too, and an operand read
outside its tensor reads the sentinel of its own guard band and poisons the result.  Misaligned twins offset valid
allocations by 1-3 floats (legal 4-byte-aligned pointers), which turns the 8-wide vector loads off; their results must be
identical to the aligned run.  Every GPU case asserts CGAN_OPT_LAST_PATH and the number of kernels launched, and the
filter-gradient table is checked to contain an unsplit case, a case capped at 512 splits and a case whose last split is
short under the device's SM count (the split rule of cgan_conv2d_wgrad_simt, restated in wgrad_splits).

Integers cannot show a loss of accumulation PRECISION (half-precision partials, or math_mode 0 quietly reaching a TF32
kernel), so a random-operand companion checks a subset of the cases, plus the kernels that cannot be made exact (batch-norm
apply / backward and the three spectral-norm entry points), against float64 with a deterministic per-element bound

    |y - y64| <= gamma(L) * A + tiny,    gamma(L) = L u / (1 - L u),  u = 2^-24,

A the same computation over absolute values and L the longest chain of dependent fp32 roundings in the kernel (derived
next to each L below from the kernel's code).  The module prints, per kernel, the number of bit-exact integer cases and the
worst err / (gamma(L) A) of the random cases.

The CPU tests check the generator and the criteria themselves, and run the case tables through tests/abi_emulator.py,
which checks the harness, the descriptors, the layouts and the guard bands without a GPU.  The emulator's torch / numpy
CPU arithmetic is bit-exact on the integer operands too, except for the batch-norm moments, which it rounds once from a
float64 mean where the kernel rounds twice: those elements are held to the gamma(L) criterion (L = 2) under the
emulator.  Only the GPU run demands bit-equality of every case."""
import ctypes
import math
import time
from fractions import Fraction

import numpy as np
import pytest
import torch

from compare_gan_b200 import _lib
from tests.abi_emulator import emulated_library, relu_gate, relu_mask, rna_tf32
from tests.test_tc_exact_gpu import contract64, out_hw

EXACT = 2 ** 24 - 1
U = 2.0 ** -24
SENTINEL = np.array([0x7FC0DEAD], np.uint32).view(np.float32)[0]      # a NaN with a payload no kernel produces
GUARD = 64                                                              # floats of guard band on each side (256 bytes)
SUMMARY = {}        # kernel -> {"exact": cases, "bound": cases, "worst": (err / (gamma(L) A), case)}


def gamma(L):
  return L * U / (1.0 - L * U)


def product_range(terms):
  """The largest R such that `terms` products of integers in [-R, R] sum below 2^24."""
  return math.isqrt(EXACT // max(terms, 1))


def cdiv(a, b):
  return -(-a // b)


def ints(rng, shape, r):
  return rng.randint(-r, r + 1, size=shape).astype(np.float32)


def record(kernel, case, ratio=None):
  s = SUMMARY.setdefault(kernel, {"exact": 0, "bound": 0, "worst": (0.0, "")})
  if ratio is None:
    s["exact"] += 1
  else:
    s["bound"] += 1
    if ratio >= s["worst"][0]:
      s["worst"] = (ratio, case)


@pytest.fixture(scope="module", autouse=True)
def _report(pytestconfig):
  t0 = time.time()
  SUMMARY.clear()
  yield
  if not SUMMARY:
    return
  lines = ["exact-fp32 kernels, %.1f s (integer cases: bit-exact; random cases: worst err / (gamma(L) A)):" % (time.time() - t0)]
  for k in sorted(SUMMARY):
    s = SUMMARY[k]
    txt = "  %-22s" % k
    if s["exact"]:
      txt += " %3d bit-exact" % s["exact"]
    if s["bound"]:
      txt += " %3d random, worst %.3e (%s)" % (s["bound"], s["worst"][0], s["worst"][1])
    lines.append(txt)
  capman = pytestconfig.pluginmanager.getplugin("capturemanager")
  tr = pytestconfig.pluginmanager.getplugin("terminalreporter")
  if capman is None or tr is None:
    print("\n".join(lines))
    return
  with capman.global_and_fixture_disabled():
    tr.ensure_newline()
    for line in lines:
      tr.write_line(line)


# ---------------------------------------------------------------------------------------------------- buffers, verdicts

def emulated(K):
  return bool(getattr(K.lib(), "emulated", False))


class Guarded(object):
  """`values` (flat float32) at float offset GUARD + misalign of a device buffer whose margins hold SENTINEL."""

  def __init__(self, K, values, misalign=0):
    values = np.ravel(np.asarray(values, np.float32))
    self.lead = GUARD + misalign
    self.initial = np.full(self.lead + values.size + GUARD, SENTINEL, np.float32)
    self.initial[self.lead:self.lead + values.size] = values
    self.dev = K.from_numpy(self.initial)
    self.ptr = self.dev.ptr + 4 * self.lead

  def read(self):
    return np.array(self.dev.cpu(), copy=True)


class HostBuf(object):
  """A Guarded look-alike holding a host array (the CPU self-tests feed verify() with it)."""

  def __init__(self, initial, lead, got):
    self.initial, self.lead, self.got = initial, lead, got

  def read(self):
    return self.got


def same(a, b):
  """Equal values, or equal bits (the sentinel NaN)."""
  return (a == b) | (a.view(np.uint32) == b.view(np.uint32))


def decode(i, shape, names):
  return ", ".join("%s=%d" % kv for kv in zip(names, np.unravel_index(int(i), shape)))


def verify(buf, offsets, expected, what, names, bound=None):
  """The whole buffer against its initial contents with `expected` written at `offsets`: the output bit-exact, every
  other float unchanged.  bound = (y64, e): an output element that is not bit-exact passes when |y - y64| <= e (the
  emulator's arithmetic, and the random-operand cases).  Returns the output values and the worst |y - y64| / e."""
  got = buf.read()
  expected = np.asarray(expected, np.float32)
  pos = buf.lead + np.asarray(offsets).ravel()
  exp = buf.initial.copy()
  exp[pos] = expected.ravel()
  bad = ~same(got, exp)
  out = got[pos].reshape(expected.shape)
  ratio = None
  if bound is not None:
    y64, e = bound
    err = np.abs(out.astype(np.float64) - y64)
    ratio = float(np.max(err / np.maximum(e, 1e-300))) if err.size else 0.0
    ok = np.isfinite(out) & (err <= e)
    bad[pos[ok.ravel()]] = False
  if bad.any():
    i = int(np.flatnonzero(bad)[0])
    k = np.flatnonzero(pos == i)
    if k.size:
      j = int(k[0])
      where = "output element (%s): got %r, expected %r" % (decode(j, expected.shape, names), float(got[i]),
                                                            float(expected.ravel()[j]))
      if bound is not None:
        where += " (float64 %r, bound %.3g)" % (float(bound[0].ravel()[j]), float(bound[1].ravel()[j]))
    else:
      where = "float %d of the buffer, outside the output (output floats %d..%d), overwritten with %r" % (
          i - buf.lead, int(pos.min()) - buf.lead, int(pos.max()) - buf.lead, float(got[i]))
    raise AssertionError("%s: %d floats differ; first at %s" % (what, int(bad.sum()), where))
  return out, ratio


def check_bound(y, y64, e, what, names):
  """|y - y64| <= e element by element; returns the worst ratio."""
  y = np.asarray(y)
  err = np.abs(y.astype(np.float64) - y64)
  bad = ~(np.isfinite(y) & (err <= e))
  if bad.any():
    j = int(np.flatnonzero(bad.ravel())[0])
    raise AssertionError("%s: %d of %d elements exceed the bound; first at (%s): got %r, float64 %r, bound %.3g" % (
        what, int(bad.sum()), y.size, decode(j, y.shape, names), float(y.ravel()[j]), float(y64.ravel()[j]),
        float(e.ravel()[j])))
  return float(np.max(err / np.maximum(e, 1e-300))) if err.size else 0.0


# ---------------------------------------------------------------------------------------------------- convolution cases

class Case(object):
  """One convolution in math_mode 0.  op: fwd (a = x, b = w), dgrad (a = dy, b = w -> dx) or wgrad (a = x, b = dy -> dw).
  kernel: the summary row; path: the CGAN_OPT_LAST_PATH the call must report.  ep: bias, residual, relu, leak (the mask
  gate), round_out.  ldy / at: the output is channels [at, at + cout) of ldy-wide pixels (cgan_conv2d_fwd_act_ld).
  twin: also run with the operands and the output 1-3 floats off their 16-byte alignment."""

  def __init__(self, kernel, path, op, n, h, w, cin, cout, kh=1, kw=1, stride=1, up=False, pad="SAME", bias=False,
               residual=False, relu=False, leak=None, round_out=False, ldy=0, at=0, twin=False, note=""):
    self.kernel, self.path, self.op = kernel, path, op
    self.n, self.h, self.w, self.cin, self.cout = n, h, w, cin, cout
    self.kh, self.kw, self.stride, self.up, self.pad = kh, kw, stride, up, pad
    self.bias, self.residual, self.relu, self.leak, self.round_out = bias, residual, relu, leak, round_out
    self.ldy, self.at, self.twin, self.note = ldy, at, twin, note

  @property
  def id(self):
    s = "%s-n%d-%dx%d-%d-%d-k%dx%d-s%d%s-%s" % (self.op, self.n, self.h, self.w, self.cin, self.cout, self.kh, self.kw,
                                               self.stride, "-up" if self.up else "", self.pad)
    for flag in ("bias", "residual", "relu"):
      if getattr(self, flag):
        s += "-" + flag
    if self.leak is not None:
      s += "-mask%g" % self.leak
    if self.round_out:
      s += "-round"
    if self.ldy:
      s += "-ldy%d@%d" % (self.ldy, self.at)
    if self.twin:
      s += "-twin"
    return s + ("-" + self.note if self.note else "")

  def out_shape(self):
    oh, ow = out_hw(self)
    return {"fwd": (self.n, oh, ow, self.cout), "dgrad": (self.n, self.h, self.w, self.cin),
            "wgrad": (self.kh, self.kw, self.cin, self.cout)}[self.op]

  def operand_shapes(self):
    oh, ow = out_hw(self)
    x, dy, w = (self.n, self.h, self.w, self.cin), (self.n, oh, ow, self.cout), (self.kh, self.kw, self.cin, self.cout)
    return {"fwd": (x, w), "dgrad": (dy, w), "wgrad": (x, dy)}[self.op]

  def terms(self):
    """Length of the contraction."""
    oh, ow = out_hw(self)
    return {"fwd": self.kh * self.kw * self.cin, "dgrad": self.kh * self.kw * self.cout, "wgrad": self.n * oh * ow}[self.op]


def gg(op, *a, **k):
  """A case for the gather-GEMM kernel (path simt_fp32)."""
  return Case("gather-gemm " + op, "simt_fp32", op, *a, **k)


def thin(kernel, op, *a, **k):
  return Case(kernel, "thin_fp32", op, *a, **k)


NAMES = {"fwd": ("n", "y", "x", "c"), "dgrad": ("n", "y", "x", "c"), "wgrad": ("kh", "kw", "ci", "co")}

GATHER_CASES = [
    # pixel counts 127 / 128 / 129 / 257 against the 128-pixel tile; cout 32 (the 32-wide column kernel), 33 (the
    # 128-wide one with 95 masked columns), 128, 129 (a one-column tail tile) and 200
    gg("fwd", 1, 1, 127, 8, 32, 3, 3, bias=True),
    gg("fwd", 2, 8, 8, 16, 33, 3, 3, bias=True, relu=True),
    gg("fwd", 1, 3, 43, 12, 129, 3, 3, bias=True, note="ktail"),              # K = 108: a 12-wide K tail, scalar loads
    gg("fwd", 1, 1, 257, 8, 128, 1, 7, bias=True, twin=True),                 # vector loads on both operands
    gg("fwd", 2, 9, 7, 8, 200, 5, 5, pad="VALID"),
    # even kernels pad asymmetrically; 1x7 / 7x1; rectangular maps
    gg("fwd", 2, 10, 6, 16, 64, 2, 2, bias=True),
    gg("fwd", 2, 9, 8, 8, 40, 4, 4, residual=True),
    gg("fwd", 2, 12, 5, 8, 32, 7, 1, bias=True),
    gg("fwd", 2, 5, 11, 5, 24, 1, 1, bias=True, note="ktail"),               # K = 5
    # stride 2 on odd maps, SAME (17 -> 9) and VALID (35 -> 17)
    gg("fwd", 2, 17, 17, 8, 48, 3, 3, stride=2, bias=True),
    gg("fwd", 1, 35, 35, 8, 32, 3, 3, stride=2, pad="VALID"),
    # the zero-inserted input, k = 3 and k = 1
    gg("fwd", 2, 6, 5, 16, 32, 3, 3, up=True, bias=True),
    gg("fwd", 2, 6, 5, 8, 48, 1, 1, up=True, bias=True),
    # the post pass (conv_post_kernel): residual, ReLU, mask, TF32 rounding
    gg("fwd", 2, 8, 8, 8, 32, 3, 3, bias=True, residual=True, relu=True, leak=0.2, round_out=True),
    gg("fwd", 2, 7, 9, 24, 33, 3, 3, leak=0.2),
    gg("fwd", 2, 7, 9, 24, 33, 3, 3, bias=True, leak=0.0, round_out=True),
    # channel slice of a wider tensor; the neighbouring channels are guarded
    gg("fwd", 2, 9, 7, 8, 36, 3, 3, bias=True, relu=True, ldy=100, at=24),
    gg("fwd", 2, 6, 7, 16, 33, 1, 1, bias=True, ldy=40, at=5),
    # cin <= 4 but cout < 16: no streaming kernel, the gather-GEMM
    gg("fwd", 2, 12, 10, 3, 8, 3, 3, bias=True),

    gg("dgrad", 1, 1, 127, 32, 16, 3, 3),
    gg("dgrad", 2, 8, 8, 33, 8, 3, 3, bias=True),
    gg("dgrad", 1, 3, 43, 129, 12, 3, 3, note="ktail"),
    gg("dgrad", 1, 1, 257, 128, 8, 1, 7, twin=True),
    gg("dgrad", 2, 8, 7, 200, 8, 5, 5, residual=True, relu=True, round_out=True),
    gg("dgrad", 2, 10, 6, 8, 16, 2, 2),
    # the transposed convolution of SNDCGAN's generator: the input gradient of a stride-2 conv, + bias
    gg("dgrad", 2, 16, 16, 16, 32, 4, 4, stride=2, bias=True, note="deconv"),
    gg("dgrad", 2, 9, 9, 8, 16, 3, 3, stride=2, pad="VALID"),
    gg("dgrad", 2, 6, 5, 16, 8, 3, 3, up=True, bias=True, leak=0.2),
    gg("dgrad", 2, 12, 10, 3, 32, 3, 3, bias=True, leak=0.0),

    gg("wgrad", 1, 4, 4, 8, 32, 3, 3, note="one-split"),
    gg("wgrad", 16, 32, 32, 8, 32, 3, 3, note="512-splits"),
    gg("wgrad", 2, 17, 17, 16, 129, 3, 3, note="short-split"),
    gg("wgrad", 2, 9, 8, 12, 33, 3, 3),
    gg("wgrad", 2, 8, 8, 16, 128, 3, 3, twin=True),
    gg("wgrad", 2, 17, 17, 8, 32, 3, 3, stride=2),
    gg("wgrad", 2, 16, 16, 16, 32, 4, 4, stride=2),
    gg("wgrad", 2, 6, 5, 8, 32, 3, 3, up=True),
    gg("wgrad", 2, 9, 11, 8, 40, 5, 5, pad="VALID"),
    gg("wgrad", 2, 7, 9, 8, 200, 2, 2),
    gg("wgrad", 2, 8, 9, 8, 16, 1, 7),
]

THIN_CASES = [
    # 1x1 over 1-4 channels: fwd_pw_thin (residual, ReLU, rounding fused; an ldy slice)
    thin("fwd_pw_thin", "fwd", 2, 9, 7, 1, 16, residual=True, relu=True),
    thin("fwd_pw_thin", "fwd", 2, 8, 5, 2, 32, bias=True),
    thin("fwd_pw_thin", "fwd", 2, 6, 7, 3, 64, bias=True, relu=True, ldy=96, at=16),
    thin("fwd_pw_thin", "fwd", 2, 5, 9, 4, 20, bias=True, round_out=True),
    # the generic streaming forward (M = kh kw cin of 25, 28, 12, 32, 3 and 12)
    thin("fwd_thin", "fwd", 2, 10, 9, 1, 16, 5, 5, bias=True),
    thin("fwd_thin", "fwd", 2, 9, 16, 4, 32, 1, 7, bias=True),
    thin("fwd_thin", "fwd", 2, 11, 7, 3, 48, 2, 2, bias=True, relu=True),
    thin("fwd_thin", "fwd", 2, 9, 10, 2, 128, 4, 4, residual=True),
    thin("fwd_thin", "fwd", 2, 6, 7, 3, 16, 1, 1, bias=True, leak=0.2, note="pw-masked"),
    thin("fwd_thin", "fwd", 2, 15, 13, 4, 24, 3, 1, stride=2, bias=True),
    # the 3x3 kernel (ReLU and rounding fused), over 1-4 channels, 16-160 output channels, upsampled and the stem shape
    thin("fwd_thin3", "fwd", 2, 9, 40, 1, 16, 3, 3, bias=True),
    thin("fwd_thin3", "fwd", 2, 7, 35, 2, 33, 3, 3, bias=True, relu=True, round_out=True),
    thin("fwd_thin3", "fwd", 2, 6, 20, 3, 128, 3, 3, up=True, bias=True),
    thin("fwd_thin3", "fwd", 2, 75, 75, 3, 32, 3, 3, stride=2, pad="VALID", bias=True, relu=True, round_out=True),
    thin("fwd_thin3", "fwd", 2, 8, 9, 4, 160, 3, 3, bias=True, residual=True),
    thin("fwd_thin3", "fwd", 2, 9, 7, 3, 64, 3, 3, bias=True, relu=True, ldy=80, at=8),
    # filter gradients: 3x3 over 1-4 channels (m = 9, 18, 27, 36), 3 output channels, 1x1; many per-CTA partials
    thin("wgrad_thin3", "wgrad", 2, 20, 20, 1, 16, 3, 3),
    thin("wgrad_thin3", "wgrad", 2, 8, 12, 2, 64, 3, 3, up=True),
    thin("wgrad_thin3", "wgrad", 4, 100, 70, 3, 128, 3, 3, note="multi-chunk"),
    thin("wgrad_thin3", "wgrad", 2, 35, 35, 4, 33, 3, 3, stride=2, pad="VALID"),
    thin("wgrad_thin_cout", "wgrad", 2, 16, 16, 16, 3, 3, 3),
    thin("wgrad_thin_cout", "wgrad", 2, 12, 20, 64, 3, 3, 3),
    thin("wgrad_pw_thin", "wgrad", 2, 16, 16, 3, 64),
]

CONV_CASES = GATHER_CASES + THIN_CASES


def wgrad_splits(c, sms):
  """(splits, k_per_split) of cgan_conv2d_wgrad_simt: enough splits to fill the SMs four times over, at most one per
  16-pixel k-tile and at most 512, then rebalanced so that every split but the last has the same number of k-tiles."""
  m, n, k = c.kh * c.kw * c.cin, c.cout, c.terms()
  tiles = cdiv(m, 128) * cdiv(n, 128 if n > 32 else 32)
  ktiles = cdiv(k, 16)
  splits = max(1, min((4 * sms + tiles - 1) // tiles, ktiles, 512))
  per = cdiv(ktiles, splits)
  return cdiv(ktiles, per), per * 16


def thin_wgrad_blocks(c, sms):
  """(blocks, longest per-block pixel chain) of cgan_wgrad_thin."""
  oh, ow = out_hw(c)
  npix = c.n * oh * ow
  if c.kernel == "wgrad_pw_thin":
    ppb = cdiv(cdiv(npix, 8 * sms // cdiv(c.cout, 128)), 8) * 8
    return cdiv(npix, ppb), ppb
  if c.kernel == "wgrad_thin3":
    nchunks = c.n * oh * cdiv(ow, 32)
    per = max(1, cdiv(nchunks, max(1, sms * 6 // cdiv(c.cout, 128))))
    return cdiv(nchunks, per), 32 * per
  ppb = cdiv(cdiv(npix, 4 * sms), 32) * 32
  return cdiv(npix, ppb), ppb


def expected_launches(c, sms):
  """Kernels the call launches (conv_dispatch.cu): the contraction, the split-K / partial reduction, the dgrad bias pass
  and the post pass (residual, mask, rounding, and for dgrad a ReLU) that the fused kernels leave out."""
  post = c.residual or c.leak is not None or c.round_out
  if c.op == "wgrad":
    return 2 if c.path == "thin_fp32" or wgrad_splits(c, sms)[0] > 1 else 1
  if c.op == "dgrad":
    return 1 + int(c.bias) + int(post or c.relu)
  if c.kernel == "fwd_pw_thin" or (c.kernel == "fwd_thin3" and not c.residual and c.leak is None):
    return 1
  return 1 + int(post)


def chain_length(c, sms):
  """L of the case: the longest chain of dependent fp32 roundings behind one output element.
  gather-GEMM: one thread accumulates its k-range with K chained FMAs (gemm.cu gather_gemm_kernel); the epilogue adds
    the bias (+1), the post pass the residual and the leak multiply (+2); split-K: k_per_split FMAs, then splitk_reduce
    adds the splits in order (+splits).
  streaming forward: M = kh kw cin chained FMAs and the bias (+1), post pass +2.
  streaming filter gradients: one CTA's pixel range (32 per chunk) of FMAs, then the partials of all CTAs (+blocks)."""
  if c.op == "wgrad" and c.path == "simt_fp32":
    splits, kps = wgrad_splits(c, sms)
    return kps + splits if splits > 1 else c.terms()
  if c.op == "wgrad":
    blocks, ppb = thin_wgrad_blocks(c, sms)
    return ppb + blocks
  return c.terms() + 3


def draw_conv(c, rng, random=False):
  sa, sb = c.operand_shapes()
  shape = c.out_shape()
  if random:
    a, b = rng.standard_normal(sa).astype(np.float32), rng.standard_normal(sb).astype(np.float32)
    r2 = 4.0
    side = lambda s: (r2 * rng.standard_normal(s)).astype(np.float32)
  else:
    r = product_range(c.terms() + int(c.bias) + int(c.residual))
    a, b = ints(rng, sa, r), ints(rng, sb, r)
    side = lambda s: ints(rng, s, r * r)
  ex = {}
  if c.bias:
    ex["bias"] = side(shape[-1])
  if c.residual:
    ex["residual"] = side(shape)
  if c.leak is not None:
    ex["mask"] = relu_mask(rng, shape)
  return a, b, ex


def conv_expected(c, a, b, ex):
  """(float32 result, float64 result, A) of the case: the contraction in float64, the epilogue on the float32 cast in
  the order of the kernels (bias, residual, ReLU, mask gate, TF32 rounding)."""
  y64 = contract64(c, a, b)
  scale = contract64(c, np.abs(a), np.abs(b))
  if "bias" in ex:
    y64 = y64 + ex["bias"].astype(np.float64)
    scale = scale + np.abs(ex["bias"].astype(np.float64))
  if "residual" in ex:
    y64 = y64 + ex["residual"]
    scale = scale + np.abs(ex["residual"].astype(np.float64))
  y = y64.astype(np.float32)
  if c.relu:
    y, y64 = np.maximum(y, np.float32(0)), np.maximum(y64, 0.0)
  if "mask" in ex:
    y = relu_gate(ex["mask"], y, c.leak)
    y64 = relu_gate(ex["mask"], y64, c.leak)
  if c.round_out:
    y = rna_tf32(y)
  return y, y64, scale


def conv_layout(c):
  """(floats of the output buffer, offset of every output element in it)."""
  shape = c.out_shape()
  if c.ldy:
    rows = int(np.prod(shape[:-1]))
    return rows * c.ldy, (np.arange(rows)[:, None] * c.ldy + c.at + np.arange(c.cout)[None, :]).reshape(shape)
  n = int(np.prod(shape))
  return n, np.arange(n).reshape(shape)


def run_conv(K, c, a, b, ex, misalign=0):
  """One call of the case's entry point; returns (output buffer, offsets, kernels launched, path)."""
  lib = K.lib()
  A, B = Guarded(K, a, misalign), Guarded(K, b, (2 * misalign) % 4)
  nbuf, offs = conv_layout(c)
  Y = Guarded(K, np.full(nbuf, SENTINEL, np.float32), (3 * misalign) % 4)
  dev = {k: K.from_numpy(v) for k, v in ex.items()}
  d = K.conv_desc(c.n, c.h, c.w, c.cin, c.cout, c.kh, c.kw, c.stride, c.up, c.pad)
  n0 = lib.launch_count()
  if c.op == "wgrad":
    K._call("conv2d_wgrad_ex", ctypes.byref(d), A.ptr, B.ptr, 0, Y.ptr)
  elif c.ldy:
    K._call("conv2d_fwd_act_ld", ctypes.byref(d), A.ptr, B.ptr, dev["bias"].ptr if "bias" in dev else None,
            K.ACT_RELU if c.relu else 0, Y.ptr + 4 * c.at, c.ldy)
  else:
    ep = K._epilogue(dev.get("bias"), dev.get("residual"), dev.get("mask"), c.leak or 0.0, c.relu, c.round_out)
    K._call("conv2d_fwd_ex" if c.op == "fwd" else "conv2d_dgrad_ex", ctypes.byref(d), A.ptr, B.ptr, ctypes.byref(ep),
            Y.ptr)
  launched = lib.launch_count() - n0
  return Y, offs, launched, _lib.PATH_NAMES[lib.get_option(_lib.OPT_LAST_PATH)]


def assert_path(K, what, path, want_path, launched, want_launches):
  if emulated(K):
    return
  assert path == want_path, "%s: ran on %s, expected %s" % (what, path, want_path)
  assert launched == want_launches, "%s: %d kernels launched, expected %d" % (what, launched, want_launches)


def check_conv_case(K, c, sms):
  rng = np.random.RandomState(seed_of(c.id))
  a, b, ex = draw_conv(c, rng)
  y, y64, scale = conv_expected(c, a, b, ex)
  Y, offs, launched, path = run_conv(K, c, a, b, ex)
  assert_path(K, c.id, path, c.path, launched, expected_launches(c, sms))
  got, _ = verify(Y, offs, y, c.id, NAMES[c.op])
  if c.twin:
    Y2, offs2, launched2, path2 = run_conv(K, c, a, b, ex, misalign=1)
    assert_path(K, c.id + " (misaligned)", path2, c.path, launched2, expected_launches(c, sms))
    got2, _ = verify(Y2, offs2, y, c.id + " (misaligned)", NAMES[c.op])
    assert np.array_equal(got.view(np.uint32), got2.view(np.uint32)), "%s: aligned and misaligned runs differ" % c.id
  if not emulated(K):
    record(c.kernel, c.id)


def seed_of(s, salt=0):
  return (sum(ord(ch) * (i + 1) for i, ch in enumerate(s)) + salt) % (2 ** 31)


# ---------------------------------------------------------------------------------------------------- GEMM cases

class Gemm(object):
  """C = alpha op(A) op(B) + beta C through cgan_gemm_batched (api "batched") or cgan_gemm.  pad: extra floats of lda,
  ldb, ldc; zero_a / zero_b: batch stride 0 (one operand broadcast over the batch); misalign: A, B and C 1-3 floats
  off their 16-byte alignment."""

  def __init__(self, ta, tb, m, n, k, batch=1, pad=(0, 0, 0), zero_a=False, zero_b=False, alpha=1.0, beta=0.0,
               misalign=0, api="batched"):
    self.ta, self.tb, self.m, self.n, self.k, self.batch = ta, tb, m, n, k, batch
    self.pad, self.zero_a, self.zero_b, self.alpha, self.beta, self.misalign, self.api = (
        pad, zero_a, zero_b, alpha, beta, misalign, api)
    assert beta == 0 or (math.frexp(alpha)[0] == 0.5 and math.frexp(beta)[0] == 0.5), "beta * C is exact for powers of 2"
    self.kernel = "gather-gemm gemm"

  @property
  def id(self):
    s = "%s-%s%s-m%d-n%d-k%d" % (self.api, "t" if self.ta else "n", "t" if self.tb else "n", self.m, self.n, self.k)
    if self.batch > 1:
      s += "-b%d" % self.batch
    if any(self.pad):
      s += "-ld+%d.%d.%d" % self.pad
    if self.zero_a or self.zero_b:
      s += "-s0" + ("a" if self.zero_a else "") + ("b" if self.zero_b else "")
    if self.alpha != 1.0 or self.beta != 0.0:
      s += "-alpha%g-beta%g" % (self.alpha, self.beta)
    if self.misalign:
      s += "-misaligned"
    return s

  def layout(self):
    ar, ac = (self.k, self.m) if self.ta else (self.m, self.k)
    br, bc = (self.n, self.k) if self.tb else (self.k, self.n)
    lda, ldb, ldc = ac + self.pad[0], bc + self.pad[1], self.n + self.pad[2]
    sa = 0 if self.zero_a else cdiv(ar * lda, 4) * 4 + 4
    sb = 0 if self.zero_b else cdiv(br * ldb, 4) * 4 + 4
    sc = self.m * ldc + 5
    return (ar, ac, lda, sa), (br, bc, ldb, sb), (ldc, sc)

  def vector_loads(self):
    """(vecA, vecB) as cgan_gemm_batched_simt decides them."""
    (_, _, lda, sa), (_, _, ldb, sb), _ = self.layout()
    return (not self.misalign and lda % 4 == 0 and sa % 4 == 0, self.misalign == 0 and ldb % 4 == 0 and sb % 4 == 0)


def G(*a, **k):
  return Gemm(*a, **k)


GEMM_CASES = [
    # the four transpose combinations at tile edges
    G(0, 0, 127, 33, 129), G(0, 1, 128, 32, 127), G(1, 0, 129, 31, 32), G(1, 1, 257, 129, 33),
    G(0, 0, 1, 1, 1), G(0, 1, 1, 257, 31), G(1, 0, 257, 1, 128), G(1, 1, 31, 128, 257),
    G(0, 0, 33, 129, 257), G(1, 1, 32, 31, 1),
    # padded leading dimensions: multiples of 4 keep the vector loads, lda % 4 != 0 turns them off
    G(0, 0, 129, 128, 64, pad=(4, 8, 3)), G(0, 1, 127, 33, 40, pad=(1, 2, 7)), G(1, 0, 64, 129, 33, pad=(3, 4, 1)),
    G(1, 1, 33, 64, 128, pad=(5, 0, 2)),
    # the same shape misaligned by 1-3 floats (vector loads off): identical to the aligned run
    G(0, 0, 129, 128, 64, pad=(4, 8, 3), misalign=1),
    # batched, with gaps between the batch items and with a broadcast operand (batch stride 0)
    G(0, 1, 33, 40, 24, batch=3, pad=(0, 0, 2)), G(0, 0, 128, 33, 31, batch=4, zero_b=True),
    G(1, 0, 31, 129, 16, batch=2, zero_a=True, pad=(1, 0, 0)), G(0, 1, 64, 64, 32, batch=3),
    # the epilogue: alpha / beta powers of two with C read, a non-power-of-two alpha (one fp32 multiply), k = 0 with
    # beta != 0 (C = beta C)
    G(0, 0, 129, 33, 65, alpha=0.5, beta=2.0), G(1, 1, 33, 129, 64, alpha=2.0, beta=0.5, pad=(0, 0, 3)),
    G(0, 1, 127, 64, 48, batch=2, alpha=0.3), G(0, 1, 31, 33, 0, beta=2.0, pad=(1, 1, 0)),
    # cgan_gemm (one matrix)
    G(0, 0, 129, 33, 127, api="gemm"), G(1, 1, 33, 200, 64, pad=(2, 1, 3), api="gemm"),
    G(0, 1, 64, 40, 32, alpha=0.5, beta=2.0, api="gemm"),
]


def gemm_operands(g, rng, random=False):
  (ar, ac, lda, sa), (br, bc, ldb, sb), (ldc, sc) = g.layout()
  na = (g.batch - 1) * sa + ar * lda if g.batch else 0
  nb = (g.batch - 1) * sb + br * ldb
  nc = (g.batch - 1) * sc + g.m * ldc
  r = product_range(g.k + (2 if g.beta else 0))
  if random:
    a, b = rng.standard_normal(max(na, 1)).astype(np.float32), rng.standard_normal(max(nb, 1)).astype(np.float32)
  else:
    a, b = ints(rng, max(na, 1), r), ints(rng, max(nb, 1), r)      # the padding holds values too: reading it fails
  c_offs = (np.arange(g.batch)[:, None, None] * sc + np.arange(g.m)[None, :, None] * ldc +
            np.arange(g.n)[None, None, :])
  c = np.full(nc, SENTINEL, np.float32)
  if g.beta:
    c[c_offs] = rng.standard_normal(c_offs.shape).astype(np.float32) if random else ints(rng, c_offs.shape, r * r)
  else:
    c[c_offs] = np.nan                      # beta = 0: C must not be read
  return a, b, c, c_offs


def gemm_views(g, a, b):
  (ar, ac, lda, sa), (br, bc, ldb, sb), _ = g.layout()
  out = []
  for i in range(g.batch):
    ai = np.lib.stride_tricks.as_strided(a[i * sa:], (ar, ac), (4 * lda, 4)).astype(np.float64)
    bi = np.lib.stride_tricks.as_strided(b[i * sb:], (br, bc), (4 * ldb, 4)).astype(np.float64)
    out.append((ai.T if g.ta else ai, bi.T if g.tb else bi))
  return out


def gemm_expected(g, a, b, c, c_offs):
  """(float32 result, float64 result, A): alpha * acc rounds once, + beta * C is exact (powers of two)."""
  prods = [(ai @ bi, np.abs(ai) @ np.abs(bi)) for ai, bi in gemm_views(g, a, b)]
  acc = np.stack([p[0] for p in prods])
  scale = np.stack([p[1] for p in prods]) * abs(g.alpha)
  c0 = c[c_offs]
  y = np.float32(g.alpha) * acc.astype(np.float32)
  y64 = g.alpha * acc
  if g.beta:
    y = y + np.float32(g.beta) * c0
    y64 = y64 + g.beta * c0.astype(np.float64)
    scale = scale + abs(g.beta) * np.abs(c0.astype(np.float64))
  return y, y64, scale


def run_gemm(K, g, a, b, c):
  lib = K.lib()
  (_, _, lda, sa), (_, _, ldb, sb), (ldc, sc) = g.layout()
  mis = g.misalign
  A, B, C = Guarded(K, a, mis), Guarded(K, b, (mis + 1) % 4 if mis else 0), Guarded(K, c, (mis + 2) % 4 if mis else 0)
  n0 = lib.launch_count()
  if g.api == "gemm":
    K._call("gemm", g.ta, g.tb, g.m, g.n, g.k, g.alpha, A.ptr, lda, B.ptr, ldb, g.beta, C.ptr, ldc)
  else:
    K._call("gemm_batched", g.ta, g.tb, g.m, g.n, g.k, g.alpha, A.ptr, lda, sa, B.ptr, ldb, sb, g.beta, C.ptr, ldc, sc,
            g.batch)
  return C, lib.launch_count() - n0, _lib.PATH_NAMES[lib.get_option(_lib.OPT_LAST_PATH)]


def check_gemm_case(K, g):
  rng = np.random.RandomState(seed_of(g.id))
  a, b, c, c_offs = gemm_operands(g, rng)
  y = gemm_expected(g, a, b, c, c_offs)[0]
  C, launched, path = run_gemm(K, g, a, b, c)
  assert_path(K, g.id, path, "simt_fp32", launched, 1)
  got, _ = verify(C, c_offs, y, g.id, ("batch", "row", "col"))
  if g.misalign:
    aligned = Gemm(g.ta, g.tb, g.m, g.n, g.k, g.batch, g.pad, g.zero_a, g.zero_b, g.alpha, g.beta, 0, g.api)
    C0 = run_gemm(K, aligned, a, b, c)[0]
    assert np.array_equal(got.view(np.uint32), C0.read()[C0.lead + c_offs].view(np.uint32)), \
        "%s: aligned and misaligned runs differ" % g.id
  if not emulated(K):
    record(g.kernel, g.id)


# ---------------------------------------------------------------------------------------------------- column reductions

class Red(object):
  """cgan_colsum over `groups` groups of `rows` rows (kind colsum) or cgan_bn_moments + cgan_bn_finalize (kind moments)."""

  def __init__(self, kind, rows, c, groups=1):
    self.kind, self.rows, self.c, self.groups = kind, rows, c, groups
    self.kernel = "colreduce " + kind

  @property
  def id(self):
    return "%s-g%d-r%d-c%d" % (self.kind, self.groups, self.rows, self.c)


RED_CASES = [
    Red("colsum", 1, 1), Red("colsum", 100000, 1), Red("colsum", 777, 31), Red("colsum", 4099, 33),
    Red("colsum", 333, 1000), Red("colsum", 37, 33, groups=256), Red("colsum", 200, 31, groups=7),
    Red("colsum", 9, 1000, groups=3),
    Red("moments", 1, 1), Red("moments", 100000, 1), Red("moments", 777, 31), Red("moments", 4099, 33),
    Red("moments", 333, 1000), Red("moments", 8, 64),
]


def colreduce_chunks(groups, rows, c, sms):
  """(chunks, rows per chunk) of norm.cu colreduce: about four CTAs per SM, at least 32 rows per chunk, a multiple of 8
  rows per chunk (the row lanes), the last chunk ragged when rows is not a multiple."""
  cblocks = cdiv(c, 32)
  want = (4 * sms + cblocks * groups - 1) // (cblocks * groups)
  chunks = max(1, min(want, cdiv(rows, 32), 65535))
  rpc = cdiv(cdiv(rows, chunks), 8) * 8
  return cdiv(rows, rpc), rpc


def colreduce_chain(groups, rows, c, sms):
  """L of colreduce: a thread adds every 8th row of its chunk (rpc / 8), 8 row lanes are added in order, the finishing
  pass adds every 8th chunk partial (chunks / 8) and its 8 lanes, and the result is scaled (+1)."""
  chunks, rpc = colreduce_chunks(groups, rows, c, sms)
  return cdiv(rpc, 8) + 8 + cdiv(chunks, 8) + 8 + 1


def round_exact_to_f32(q):
  """The float32 nearest to the rational q (ties to even)."""
  f = np.float32(float(q))
  cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
  best = min(cands, key=lambda v: (abs(Fraction(float(v)) - q), int(np.array(v, np.float32).view(np.uint32)) & 1))
  return np.float32(best)


def check_red_case(K, rc):
  lib = K.lib()
  rng = np.random.RandomState(seed_of(rc.id))
  total = rc.groups * rc.rows
  if rc.kind == "colsum":
    r = EXACT // rc.rows
    x = ints(rng, (total, rc.c), min(r, 1 << 20))
    out, xd = Guarded(K, np.full(rc.groups * rc.c, SENTINEL, np.float32)), K.from_numpy(x)
    n0 = lib.launch_count()
    K._call("colsum", out.ptr, xd.ptr, rc.groups, rc.rows, rc.c)
    assert_path(K, rc.id, "simt_fp32", "simt_fp32", lib.launch_count() - n0, 1)
    xs = x.reshape(rc.groups, rc.rows, rc.c).astype(np.float64)
    verify(out, np.arange(rc.groups * rc.c).reshape(rc.groups, rc.c), xs.sum(1).astype(np.float32), rc.id,
           ("group", "c"))
  else:
    x = ints(rng, (rc.rows, rc.c), product_range(rc.rows))
    xd = K.from_numpy(x)
    stats = Guarded(K, np.full(2 * rc.c, SENTINEL, np.float32))
    n0 = lib.launch_count()
    K._call("bn_moments", stats.ptr, xd.ptr, rc.rows, rc.c)
    assert_path(K, rc.id, "simt_fp32", "simt_fp32", lib.launch_count() - n0, 1)
    xs = x.astype(np.float64)
    s1, s2 = xs.sum(0), (xs * xs).sum(0)          # exact integers below 2^24
    scale = np.float32(1.0) / np.float32(rc.rows)   # the kernel multiplies by 1.0f / rows
    want = np.concatenate([s1.astype(np.float32) * scale, s2.astype(np.float32) * scale])
    # the emulator rounds the float64 mean once where the kernel rounds the sum and the product by 1 / rows (L = 2)
    bound = None
    if emulated(K):
      bound = (np.concatenate([s1, s2]) / rc.rows, gamma(2) * np.concatenate([np.abs(xs).sum(0), s2]) / rc.rows)
    got, _ = verify(stats, np.arange(2 * rc.c), want, rc.id, ("stat",), bound)
    # bn_finalize: var = msq - mean * mean, which nvcc may contract into one FMA (one rounding of the exact value) or
    # evaluate as a rounded product and a rounded difference: either rounding is accepted, element by element
    mv = Guarded(K, np.full(2 * rc.c, SENTINEL, np.float32))
    K._call("bn_finalize", mv.ptr, stats.ptr, rc.c, None, None, 0.0)
    res = mv.read()[mv.lead:mv.lead + 2 * rc.c]
    mean, msq = got[:rc.c], got[rc.c:]
    assert np.array_equal(res[:rc.c].view(np.uint32), mean.view(np.uint32)), "%s: finalize mean" % rc.id
    separate = (msq - (mean * mean).astype(np.float32)).astype(np.float32)
    fused = np.array([round_exact_to_f32(Fraction(float(q)) - Fraction(float(m)) ** 2) for m, q in zip(mean, msq)],
                     np.float32)
    ok = same(res[rc.c:], separate) | same(res[rc.c:], fused)
    assert ok.all(), "%s: finalize var at c=%d: %r is neither %r (separate) nor %r (fused)" % (
        rc.id, int(np.flatnonzero(~ok)[0]), float(res[rc.c:][~ok][0]), float(separate[~ok][0]), float(fused[~ok][0]))
    assert np.array_equal(mv.read()[:mv.lead].view(np.uint32), mv.initial[:mv.lead].view(np.uint32))
    assert np.array_equal(mv.read()[mv.lead + 2 * rc.c:].view(np.uint32), mv.initial[mv.lead + 2 * rc.c:].view(np.uint32))
  if not emulated(K):
    record(rc.kernel, rc.id)


# ---------------------------------------------------------------------------------------------------- fixtures, GPU tests

@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  kernels.set_math_mode(0)
  return kernels


@pytest.fixture(scope="module")
def sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("c", CONV_CASES, ids=[c.id for c in CONV_CASES])
def test_conv_integer_operands_bit_exact(K, sms, c):
  check_conv_case(K, c, sms)


@pytest.mark.gpu
@pytest.mark.parametrize("g", GEMM_CASES, ids=[g.id for g in GEMM_CASES])
def test_gemm_integer_operands_bit_exact(K, g):
  check_gemm_case(K, g)


@pytest.mark.gpu
@pytest.mark.parametrize("rc", RED_CASES, ids=[r.id for r in RED_CASES])
def test_column_reductions_bit_exact(K, rc):
  check_red_case(K, rc)


@pytest.mark.gpu
def test_reduction_ticket_counters_reset_themselves(K):
  """The single-launch colreduce hands the finishing pass to the last CTA of each column block through a ticket counter,
  which that CTA resets: the same call twice in a row, then interleaved with other shapes, stays exact every time
  (a counter left non-zero would leave the output at its sentinel or finish early)."""
  a, b, c = Red("colsum", 4099, 33), Red("moments", 777, 31), Red("colsum", 37, 33, groups=256)
  for rc in (a, a, b, a, c, b, c, a):
    check_red_case(K, rc)


@pytest.mark.gpu
def test_case_tables_cover_the_kernel_branches(sms):
  """On this GPU's SM count the filter-gradient table holds an unsplit case, a case capped at 512 splits (possible only
  when 4 x SMs > 512) and a case whose last split is short; the tables reach both column kernels, K tails, vector and
  scalar loads, and ragged / many-chunk reductions."""
  check_tables(sms)


def check_tables(sms):
  simt_w = [c for c in GATHER_CASES if c.op == "wgrad"]
  splits = {c.id: wgrad_splits(c, sms) for c in simt_w}
  assert any(s == 1 for s, _ in splits.values()), splits
  if 4 * sms > 512:
    assert any(s == 512 for s, _ in splits.values()), splits
  assert any(s > 1 and c.terms() - (s - 1) * kps < kps for c in simt_w for s, kps in [splits[c.id]]), splits
  cols = [c.cout if c.op != "dgrad" else c.cin for c in GATHER_CASES]
  assert {32, 33, 128, 129, 200} <= set(cols)
  pixels = {c.n * out_hw(c)[0] * out_hw(c)[1] for c in GATHER_CASES if c.op == "fwd"}
  assert {127, 128, 129, 257} <= pixels
  assert any(c.terms() % 16 for c in GATHER_CASES if c.op != "wgrad")
  assert any(c.cin % 8 == 0 and c.cout % 8 == 0 and c.twin for c in GATHER_CASES)
  assert any(c.cin % 8 and c.op == "fwd" for c in GATHER_CASES)
  vec = [g.vector_loads() for g in GEMM_CASES]
  assert (True, True) in vec and any(not a for a, _ in vec)
  chunks = [colreduce_chunks(r.groups, r.rows, r.c, sms) for r in RED_CASES]
  assert any(r.rows % rpc for r, (_, rpc) in zip(RED_CASES, chunks))
  assert any(n > 8 for n, _ in chunks)
  assert max(r.groups for r in RED_CASES) == 256
  assert {1, 31, 33, 1000} <= {r.c for r in RED_CASES}
  thin_w = [c for c in THIN_CASES if c.kernel == "wgrad_thin3"]
  assert {9, 18, 27, 36} <= {9 * c.cin for c in thin_w}
  assert any(thin_wgrad_blocks(c, sms)[1] > 32 for c in thin_w)


# ---------------------------------------------------------------------------------------------------- random operands

RANDOM_CONV = [
    gg("fwd", 1, 3, 43, 12, 129, 3, 3, bias=True, note="ktail"),
    gg("fwd", 2, 9, 8, 8, 40, 4, 4, residual=True),
    gg("fwd", 2, 7, 9, 24, 33, 3, 3, bias=True, relu=True, leak=0.2),
    gg("dgrad", 2, 16, 16, 16, 32, 4, 4, stride=2, bias=True, note="deconv"),
    gg("dgrad", 1, 1, 257, 128, 8, 1, 7),
    gg("wgrad", 16, 32, 32, 8, 32, 3, 3, note="512-splits"),
    gg("wgrad", 2, 17, 17, 16, 129, 3, 3, note="short-split"),
    gg("wgrad", 1, 4, 4, 8, 32, 3, 3, note="one-split"),
    thin("fwd_pw_thin", "fwd", 2, 9, 7, 1, 16, residual=True, relu=True),
    thin("fwd_thin", "fwd", 2, 9, 10, 2, 128, 4, 4, residual=True),
    thin("fwd_thin3", "fwd", 2, 8, 9, 4, 160, 3, 3, bias=True, residual=True),
    thin("wgrad_thin3", "wgrad", 4, 100, 70, 3, 128, 3, 3, note="multi-chunk"),
    thin("wgrad_thin_cout", "wgrad", 2, 12, 20, 64, 3, 3, 3),
    thin("wgrad_pw_thin", "wgrad", 2, 16, 16, 3, 64),
]

RANDOM_GEMM = [G(1, 1, 257, 129, 33), G(0, 0, 33, 129, 257), G(0, 1, 127, 64, 48, batch=2, alpha=0.3),
               G(0, 0, 129, 33, 65, alpha=0.5, beta=2.0)]


def check_random_conv(K, c, sms):
  rng = np.random.RandomState(seed_of(c.id, 11))
  a, b, ex = draw_conv(c, rng, random=True)
  _, y64, scale = conv_expected(c, a, b, ex)
  Y, offs, launched, path = run_conv(K, c, a, b, ex)
  assert_path(K, c.id, path, c.path, launched, expected_launches(c, sms))
  _, ratio = verify(Y, offs, np.zeros(y64.shape, np.float32), c.id + " (random)", NAMES[c.op],
                    (y64, gamma(chain_length(c, sms)) * scale + 1e-30))
  return ratio


def check_random_gemm(K, g):
  rng = np.random.RandomState(seed_of(g.id, 11))
  a, b, c, c_offs = gemm_operands(g, rng, random=True)
  _, y64, scale = gemm_expected(g, a, b, c, c_offs)
  C, launched, path = run_gemm(K, g, a, b, c)
  assert_path(K, g.id, path, "simt_fp32", launched, 1)
  # L: k chained FMAs, the alpha multiply and the beta * C addition
  _, ratio = verify(C, c_offs, np.zeros(y64.shape, np.float32), g.id + " (random)", ("batch", "row", "col"),
                    (y64, gamma(g.k + 2) * scale + 1e-30))
  return ratio


@pytest.mark.gpu
@pytest.mark.parametrize("c", RANDOM_CONV, ids=[c.id for c in RANDOM_CONV])
def test_conv_random_operands_within_fp32_bound(K, sms, c):
  record(c.kernel, c.id, check_random_conv(K, c, sms))


@pytest.mark.gpu
@pytest.mark.parametrize("g", RANDOM_GEMM, ids=[g.id for g in RANDOM_GEMM])
def test_gemm_random_operands_within_fp32_bound(K, g):
  record(g.kernel, g.id, check_random_gemm(K, g))


# batch norm -----------------------------------------------------------------------------------------------------------

def bn_inputs(rng, rows, c):
  x = (3.0 * rng.standard_normal((rows, c)) + 1.0).astype(np.float32)
  mean = x.astype(np.float64).mean(0).astype(np.float32)
  var = x.astype(np.float64).var(0).astype(np.float32)
  return x, np.concatenate([mean, var]), rng.standard_normal(c).astype(np.float32), rng.standard_normal(c).astype(np.float32)


def check_bn(K, rows, c, sms, relu=False):
  """bn_apply, bn_bwd_reduce and bn_bwd_apply (cond = 0) on random operands; returns the worst ratios."""
  rng = np.random.RandomState(seed_of("bn%d-%d" % (rows, c)))
  x, mv, gam, bet = bn_inputs(rng, rows, c)
  dy = rng.standard_normal((rows, c)).astype(np.float32)
  eps = 1e-5
  X, MV, GA, BE, DY = (K.from_numpy(v) for v in (x, mv, gam, bet, dy))
  mean, var = mv[:c].astype(np.float64), mv[c:].astype(np.float64)
  inv = 1.0 / np.sqrt(var + np.float64(np.float32(eps)))
  x64, g64 = x.astype(np.float64), gam.astype(np.float64)
  xh, axh = (x64 - mean) * inv, (np.abs(x64) + np.abs(mean)) * inv
  names = ("row", "c")
  ratios = {}
  # apply: L = 7 (var + eps, sqrt, reciprocal, x - mean, * inv, * gamma, + beta)
  y = Guarded(K, np.full(rows * c, SENTINEL, np.float32))
  K._call("bn_apply", y.ptr, X.ptr, rows, c, rows, MV.ptr, eps, GA.ptr, BE.ptr, 0, 1 if relu else 0)
  y64 = xh * g64 + bet
  if relu:
    y64 = np.maximum(y64, 0.0)
  e = gamma(7) * (axh * np.abs(g64) + np.abs(bet)) + 1e-30
  ratios["bn_apply"] = verify(y, np.arange(rows * c).reshape(rows, c), np.zeros((rows, c), np.float32), "bn_apply",
                              names, (y64, e))[1]
  # backward reduction: per row 6 roundings (inv: 3, x - mean, * inv, dy * xhat), the colreduce chain, then * gamma
  L = colreduce_chain(1, rows, c, sms) + 7
  sums, dgam, dbet = (Guarded(K, np.full(n, SENTINEL, np.float32)) for n in (2 * c, c, c))
  K._call("bn_bwd_reduce", sums.ptr, dgam.ptr, dbet.ptr, DY.ptr, X.ptr, rows, c, rows, MV.ptr, eps, GA.ptr, 0)
  dy64 = dy.astype(np.float64)
  dg64, adg = (dy64 * xh).sum(0), (np.abs(dy64) * axh).sum(0)
  db64, adb = dy64.sum(0), np.abs(dy64).sum(0)
  ar = np.arange(c)
  r1 = verify(dgam, ar, np.zeros(c, np.float32), "bn_bwd_reduce dgamma", ("c",), (dg64, gamma(L) * adg + 1e-30))[1]
  r2 = verify(dbet, ar, np.zeros(c, np.float32), "bn_bwd_reduce dbeta", ("c",), (db64, gamma(L) * adb + 1e-30))[1]
  s64 = np.concatenate([g64 * db64, g64 * dg64])
  sa = np.concatenate([np.abs(g64) * adb, np.abs(g64) * adg])
  got, r3 = verify(sums, np.arange(2 * c), np.zeros(2 * c, np.float32), "bn_bwd_reduce sums", ("i",),
                   (s64, gamma(L) * sa + 1e-30))
  ratios["bn_bwd_reduce"] = max(r1, r2, r3)
  # backward apply on the sums the GPU produced: L = 12 (inv: 3, xhat: 2, dy * gamma, two products by 1 / count, the
  # xhat * s2 product, two subtractions, * inv)
  S = K.from_numpy(got)
  ic = np.float32(1.0) / np.float32(rows)
  dx = Guarded(K, np.full(rows * c, SENTINEL, np.float32))
  K._call("bn_bwd_apply", dx.ptr, DY.ptr, X.ptr, rows, c, rows, MV.ptr, eps, GA.ptr, 0, S.ptr, float(ic), 0)
  s1, s2, ic64 = got[:c].astype(np.float64), got[c:].astype(np.float64), float(ic)
  dx64 = inv * (dy64 * g64 - s1 * ic64 - xh * s2 * ic64)
  e = gamma(12) * inv * (np.abs(dy64 * g64) + np.abs(s1) * ic64 + axh * np.abs(s2) * ic64) + 1e-30
  ratios["bn_bwd_apply"] = verify(dx, np.arange(rows * c).reshape(rows, c), np.zeros((rows, c), np.float32),
                                  "bn_bwd_apply", names, (dx64, e))[1]
  return ratios


@pytest.mark.gpu
@pytest.mark.parametrize("rows,c,relu", [(1000, 33, False), (1000, 64, True), (4099, 1, False)],
                         ids=["r1000-c33-scalar", "r1000-c64-float4-relu", "r4099-c1"])
def test_batch_norm_random_operands_within_fp32_bound(K, sms, rows, c, relu):
  for k, r in check_bn(K, rows, c, sms, relu).items():
    record(k, "r%d-c%d" % (rows, c), r)


# spectral norm --------------------------------------------------------------------------------------------------------

def normalize_bound(t, e_t, n):
  """v = t / ||t|| and its first-order error bound from errors e_t in t, plus the normalisation itself: the sum of
  squares (a block-wide sum: n / 1024 per thread and two 5-level shuffle trees), the square root, the reciprocal and the
  multiply."""
  nt = np.linalg.norm(t)
  v = t / nt
  return v, (e_t + np.abs(v) * np.linalg.norm(e_t)) / nt + gamma(cdiv(n, 1024) + 14) * np.abs(v)


def sn_reference(w, u, left):
  """arch_ops.py:503-531 in float64 from the same u, with per-element error bounds of an fp32 evaluation.  Every dot
  product of length n is bounded with L = n + 32, which covers each summation tree the kernels use (sn_coldot: rows /
  lanes per thread then up to 32 lanes, or all rows in one chain when lanes = 1; sn_rowdot / gemv_rows: cols / 32 per lane
  and a 5-level shuffle tree; the colreduce chain of gemv_cols)."""
  W = w.astype(np.float64)
  M = W if left else W.T                       # left: v = normalize(W^T u), u' = normalize(W v); right: the transpose
  u64 = u.astype(np.float64)
  t = M.T @ u64
  e_t = gamma(M.shape[0] + 32) * (np.abs(M).T @ np.abs(u64))
  v, e_v = normalize_bound(t, e_t, t.size)
  s = M @ v
  e_s = gamma(M.shape[1] + 32) * (np.abs(M) @ np.abs(v)) + np.abs(M) @ e_v
  un, e_u = normalize_bound(s, e_s, s.size)
  sigma = np.linalg.norm(s)
  e_sigma = np.linalg.norm(e_s) + gamma(cdiv(s.size, 1024) + 14) * sigma
  wbar = W / sigma
  e_wbar = np.abs(W) * e_sigma / sigma ** 2 + gamma(2) * np.abs(wbar)
  return {"v": (v, e_v + 1e-30), "u": (un, e_u + 1e-30), "sigma": (np.array([sigma]), np.array([e_sigma])),
          "wbar": (wbar, e_wbar + 1e-30)}


SN_ITEMS = [
    # (rows, cols, left): cols < 32, cols not a power of two, several 1024-column blocks, rows + cols > 11264 (the
    # shared-memory vectors exceed 48 KB)
    (7, 20, 1), (9, 20, 0), (27, 1000, 1), (30, 1000, 0), (20, 1536, 1), (16, 4096, 0), (1152, 96, 1), (64, 11300, 1),
    (11300, 40, 0),
]


def sn_item_data(i, rows, cols, left):
  rng = np.random.RandomState(seed_of("sn-%d-%d-%d-%d" % (i, rows, cols, left)))
  w = (rng.standard_normal((rows, cols)) / math.sqrt(rows)).astype(np.float32)
  u = rng.standard_normal(rows if left else cols).astype(np.float32)
  return w, u


def run_sn_batched(K, items):
  """One cgan_spectral_norm_batched launch over `items` [(rows, cols, left, w, u)]; returns per item {name: values}."""
  recs = np.zeros(len(items), dtype=[("w", "<u8"), ("u", "<u8"), ("rows", "<i4"), ("cols", "<i4"), ("left", "<i4"),
                                     ("reserved", "<i4"), ("wbar_off", "<i8"), ("v_off", "<i8"), ("u_off", "<i8")])
  keep, layout = [], []
  wo = vo = uo = 0
  for i, (rows, cols, left, w, u) in enumerate(items):
    W, Ub = K.from_numpy(w), Guarded(K, u)
    keep += [W, Ub]
    nu, nv = (rows, cols) if left else (cols, rows)
    recs[i] = (W.ptr, Ub.ptr, rows, cols, left, 0, wo, vo, uo)
    layout.append((Ub, wo, vo, uo, nu, nv))
    wo, vo, uo = wo + rows * cols + 3, vo + nv + 5, uo + nu + 7          # gaps between the items stay guarded
  table = K.from_numpy(recs.view(np.uint8))
  wbar, vb, ub = (Guarded(K, np.full(n, SENTINEL, np.float32)) for n in (wo, vo, uo))
  sig = Guarded(K, np.full(len(items), SENTINEL, np.float32))
  lib = K.lib()
  n0 = lib.launch_count()
  K._call("spectral_norm_batched", table.ptr, len(items), max(r + c for r, c, _, _, _ in items), 1e-12, wbar.ptr, vb.ptr,
          sig.ptr, ub.ptr)
  assert_path(K, "sn batched", "simt_fp32", "simt_fp32", lib.launch_count() - n0, 1)
  out = []
  bufs = [b.read() for b in (wbar, vb, ub, sig)]
  for i, ((rows, cols, left, w, u), (Ub, o_w, o_v, o_u, nu, nv)) in enumerate(zip(items, layout)):
    out.append({"wbar": bufs[0][wbar.lead + o_w:wbar.lead + o_w + rows * cols].reshape(rows, cols),
                "v": bufs[1][vb.lead + o_v:vb.lead + o_v + nv], "u_used": bufs[2][ub.lead + o_u:ub.lead + o_u + nu],
                "sigma": bufs[3][sig.lead + i:sig.lead + i + 1], "u": Ub.read()[Ub.lead:Ub.lead + nu]})
    assert_guards(Ub, nu, "sn item %d u" % i)
  # everything between and around the items keeps its sentinel
  for buf, spans in ((wbar, [(l[1], r * c) for l, (r, c, _, _, _) in zip(layout, items)]),
                     (vb, [(l[2], l[5]) for l in layout]), (ub, [(l[3], l[4]) for l in layout])):
    got = buf.read()
    mask = np.ones(got.size, bool)
    for off, n in spans:
      mask[buf.lead + off:buf.lead + off + n] = False
    assert np.array_equal(got[mask].view(np.uint32), buf.initial[mask].view(np.uint32)), "sn batched: guard overwritten"
  return out


def assert_guards(buf, n, what):
  got = buf.read()
  assert np.array_equal(got[:buf.lead].view(np.uint32), buf.initial[:buf.lead].view(np.uint32)), what
  assert np.array_equal(got[buf.lead + n:].view(np.uint32), buf.initial[buf.lead + n:].view(np.uint32)), what


def run_sn_single(K, rows, cols, left, w, u):
  Ub = Guarded(K, u)
  nv = cols if left else rows
  v, sig, wbar = (Guarded(K, np.full(n, SENTINEL, np.float32)) for n in (nv, 1, rows * cols))
  W = K.from_numpy(w)
  K._call("spectral_norm", W.ptr, rows, cols, left, 1e-12, Ub.ptr, v.ptr, sig.ptr, wbar.ptr)
  res = {}
  for name, buf, n in (("u", Ub, u.size), ("v", v, nv), ("sigma", sig, 1), ("wbar", wbar, rows * cols)):
    assert_guards(buf, n, "spectral_norm " + name)
    res[name] = buf.read()[buf.lead:buf.lead + n]
  res["wbar"] = res["wbar"].reshape(rows, cols)
  return res


def check_sn(K, items):
  """The batched launch over `items` (indices into SN_ITEMS) against float64 and against the per-weight entry point;
  returns the worst ratio."""
  data = [SN_ITEMS[i] + sn_item_data(i, *SN_ITEMS[i]) for i in items]
  batched = run_sn_batched(K, data)
  worst = 0.0
  for i, (rows, cols, left, w, u), got in zip(items, data, batched):
    what = "sn item %d (%dx%d, %s)" % (i, rows, cols, "left" if left else "right")
    ref = sn_reference(w, u, left)
    assert np.array_equal(got["u"].view(np.uint32), got["u_used"].view(np.uint32)), what + ": u and u_used differ"
    single = run_sn_single(K, rows, cols, left, w, u)
    for name in ("v", "u", "sigma", "wbar"):
      y64, e = ref[name]
      worst = max(worst, check_bound(got[name], y64, e, what + " batched " + name, ("i", "j")[:y64.ndim]))
      check_bound(single[name], y64, e, what + " per-weight " + name, ("i", "j")[:y64.ndim])
      # both within the bound of float64, so within twice of each other
      check_bound(got[name], single[name].astype(np.float64), 2 * e, what + " batched vs per-weight " + name,
                  ("i", "j")[:y64.ndim])
  return worst, batched


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(SN_ITEMS)), ids=["%dx%d-%s" % (r, c, "left" if l else "right")
                                                          for r, c, l in SN_ITEMS])
def test_spectral_norm_batched_items(K, i):
  record("sn batched", "item %d" % i, check_sn(K, [i])[0])


@pytest.mark.gpu
def test_spectral_norm_batched_mixed_launch(K):
  """Every item in ONE launch (shared memory sized for the largest): each item bit-identical to its own launch."""
  mixed_worst, mixed = check_sn(K, list(range(len(SN_ITEMS))))
  record("sn batched", "mixed launch", mixed_worst)
  for i in range(len(SN_ITEMS)):
    alone = check_sn(K, [i])[1][0]
    for name in ("v", "u", "sigma", "wbar", "u_used"):
      assert np.array_equal(mixed[i][name].view(np.uint32), alone[name].view(np.uint32)), \
          "item %d: %s differs between the mixed and the single launch" % (i, name)


def check_sn_bwd(K, rows, cols, left):
  """cgan_spectral_norm_bwd: dw = (dwbar - <dwbar, wbar> outer) / sigma.  The dot product of n = rows cols terms is
  bounded with L = n (every summation tree of n products), then outer (1), dp * outer (1), the subtraction (1), the
  reciprocal of sigma (1) and the multiply (1)."""
  rng = np.random.RandomState(seed_of("snbwd-%d-%d-%d" % (rows, cols, left)))
  w, u = sn_item_data(0, rows, cols, left)
  res = run_sn_single(K, rows, cols, left, w, u)
  dwbar = rng.standard_normal((rows, cols)).astype(np.float32)
  dw = Guarded(K, np.full(rows * cols, SENTINEL, np.float32))
  G_, WB, U_, V_, S_ = (K.from_numpy(v) for v in (dwbar, res["wbar"], res["u"], res["v"], res["sigma"]))
  K._call("spectral_norm_bwd", dw.ptr, G_.ptr, WB.ptr, rows, cols, left, U_.ptr, V_.ptr, S_.ptr)
  g, wb = dwbar.astype(np.float64), res["wbar"].astype(np.float64)
  uu, vv, s = res["u"].astype(np.float64), res["v"].astype(np.float64), float(res["sigma"][0])
  outer = np.outer(uu, vv) if left else np.outer(vv, uu)
  dp, adp = (g * wb).sum(), np.abs(g * wb).sum()
  y64 = (g - dp * outer) / s
  e = (gamma(5) * (np.abs(g) + abs(dp) * np.abs(outer)) + gamma(rows * cols) * adp * np.abs(outer)) / s + 1e-30
  return verify(dw, np.arange(rows * cols).reshape(rows, cols), np.zeros((rows, cols), np.float32), "spectral_norm_bwd",
                ("r", "c"), (y64, e))[1]


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols,left", [(27, 1000, 1), (300, 64, 0)], ids=["27x1000-left", "300x64-right"])
def test_spectral_norm_backward_within_fp32_bound(K, rows, cols, left):
  record("sn bwd", "%dx%d" % (rows, cols), check_sn_bwd(K, rows, cols, left))


# ---------------------------------------------------------------------------------------------------- CPU tests

def test_integer_generator_and_exact_criterion():
  """The generator keeps every partial sum below 2^24 for every case of the tables (so any summation order is exact:
  a float32 sequential sum equals float64, forwards and backwards), and assert-equality fails for one dropped term at
  one element and for a tap shifted by one pixel."""
  for c in CONV_CASES:
    a, b, ex = draw_conv(c, np.random.RandomState(seed_of(c.id)))
    _, _, scale = conv_expected(c, a, b, ex)
    assert scale.max() <= EXACT, (c.id, scale.max())
  for g in GEMM_CASES:
    a, b, cc, offs = gemm_operands(g, np.random.RandomState(seed_of(g.id)))
    _, _, scale = gemm_expected(g, a, b, cc, offs)
    assert scale.size == 0 or scale.max() <= EXACT, (g.id, scale.max())
  # sequential float32 sums in both orders equal float64
  g = Gemm(0, 0, 40, 30, 4096)
  r = product_range(g.k)
  rng = np.random.RandomState(1)
  a, b = ints(rng, (g.m, g.k), r), ints(rng, (g.k, g.n), r)
  y64 = a.astype(np.float64) @ b.astype(np.float64)
  for order in (range(g.k), reversed(range(g.k))):
    acc = np.zeros((g.m, g.n), np.float32)
    for k in order:
      acc += a[:, k:k + 1] * b[k:k + 1, :]
    assert np.array_equal(acc, y64.astype(np.float32))
  # defects
  c = gg("fwd", 2, 9, 8, 8, 40, 3, 3, bias=True)
  a, b, ex = draw_conv(c, np.random.RandomState(seed_of(c.id)))
  y, _, _ = conv_expected(c, a, b, ex)
  offs = np.arange(y.size).reshape(y.shape)
  initial = np.full(2 * GUARD + y.size, SENTINEL, np.float32)

  def host(out):
    got = initial.copy()
    got[GUARD:GUARD + y.size] = out.ravel()
    return HostBuf(initial, GUARD, got)
  verify(host(y), offs, y, "self", NAMES["fwd"])
  t = y.copy()
  t[1, 0, 3, 5] -= a[1, 0, 3, 2] * b[1, 1, 2, 5] or 1.0           # one product of the centre tap
  with pytest.raises(AssertionError, match=r"n=1, y=0, x=3, c=5"):
    verify(host(t), offs, y, "dropped term", NAMES["fwd"])
  shifted = a.copy()
  shifted[:, :, 1:] = a[:, :, :-1]
  with pytest.raises(AssertionError):
    verify(host(conv_expected(c, shifted, b, ex)[0]), offs, y, "tap shifted by one pixel", NAMES["fwd"])
  stray = host(y)
  stray.got[GUARD + y.size + 2] = 0.0
  with pytest.raises(AssertionError, match="outside the output"):
    verify(stray, offs, y, "stray write", NAMES["fwd"])


def test_gamma_criterion_accepts_fp32_and_rejects_one_dropped_term():
  """gamma(L) A accepts a float32 sequential sum of L terms and rejects the same sum with its largest term dropped,
  on a case where that term exceeds the bound."""
  L = 4096
  x = np.random.RandomState(3).standard_normal(L).astype(np.float32)
  acc = np.float32(0)
  for v in x:
    acc = np.float32(acc + v)
  y64, A = x.astype(np.float64).sum(), np.abs(x.astype(np.float64)).sum()
  e = np.array([gamma(L) * A])
  check_bound(np.array([acc]), np.array([y64]), e, "fp32 sum", ("i",))
  j = int(np.argmax(np.abs(x)))
  assert abs(x[j]) > e[0]
  with pytest.raises(AssertionError):
    check_bound(np.array([acc - x[j]]), np.array([y64]), e, "one term dropped", ("i",))


def test_case_tables_and_split_rule_on_132_sms():
  check_tables(132)


def test_case_tables_on_the_emulator():
  """Every table through tests/abi_emulator.py: descriptors, layouts, guard bands and references agree with the C-ABI's
  contract on the CPU.  Path and launch assertions are specific to the library and skipped; where the emulator's CPU
  arithmetic is not bit-exact the gamma(L) criterion applies (module docstring)."""
  from compare_gan_b200 import kernels
  with emulated_library():
    kernels.set_math_mode(0)
    for c in CONV_CASES:
      if c.n * c.h * c.w > 20000:
        continue            # the 28000-pixel filter gradient: minutes of per-pixel emulation for no extra coverage
      check_conv_case(kernels, c, 132)
    for g in GEMM_CASES:
      check_gemm_case(kernels, g)
    for rc in RED_CASES:
      check_red_case(kernels, rc)
    for c in RANDOM_CONV[:4]:
      check_random_conv(kernels, c, 132)
    for g in RANDOM_GEMM:
      check_random_gemm(kernels, g)
    check_bn(kernels, 1000, 33, 132)
    check_sn(kernels, [0, 1, 2, 3, 6])
    check_sn_bwd(kernels, 27, 1000, 1)
