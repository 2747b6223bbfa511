"""The tensor-core contractions of math_mode 1 (csrc/conv_tc.cu, thin_tc.cu, wgrad_tc.cu and the batched GEMM that
conv_dispatch.cu routes onto them), element by element against float64.

Every case draws seeded operands that are exactly representable in TF32.  Each product the tensor cores form is then
exact in fp32, and the only error left is fp32 accumulation.  The verdict is per element:

    |y - y64| <= TAU * A + 1e-30,    A = the same contraction over |operands|  (+ |bias| + |residual|)

with y64 the contraction in float64 on the CPU.  A wrong tap, offset, phase, tile mask or epilogue at one pixel fails
here instead of vanishing in a whole-tensor norm: one missing 8-channel k-step of one tap moves err / A by about
sqrt(8) / (0.64 K), 1e-3 at K = 4608, while fp32 accumulation stays orders of magnitude below TAU
(test_criterion_accepts_fp32_and_rejects_local_defects shows both on the CPU).

Beside that criterion the file pins what must hold bit for bit (the fused epilogues against y0 computed without them,
the pre-rounded operand flags, one vs two pixel tiles per CTA, two runs of every case) and the operand rounding mode of
every path: round to nearest, ties away from zero (cvt.rna), checked with operands whose low 13 bits sit at or next to a
rounding tie.  Each GPU case asserts that the tensor-core path ran (and, where the code fixes it, how many kernels were
launched), so a dispatch change cannot move it to the exact-fp32 kernels unnoticed.  Cases meant for one conv kernel
variant (a column-tile width, two pixel tiles per CTA, the halo kernel) also assert the geometry the launch reports
through CGAN_OPT_LAST_TC_BN / _MT / _HALO, so a change of the tiling rules cannot quietly empty them.

Two tests run without a GPU: the criterion's self-test, and the element-wise cases against tests/abi_emulator.py."""
import ctypes
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from compare_gan_b200 import _lib
from tests.abi_emulator import emulated_library, relu_gate, relu_mask, rna_tf32

TAU = 1e-4
WORST = {}          # path -> (worst err / A, case) of this session; printed when the module finishes


# ---------------------------------------------------------------------------------------------------- cases

class Case(object):
  """One contraction.  op: fwd (a = x, b = w), dgrad (a = dy, b = w -> dx) or wgrad (a = x, b = dy -> dw); bmm_nt /
  bmm_nn / bmm_tn (a, b the batched matrices).  ep: bias, residual, relu, leak (a float: the (leaky-)ReLU mask gate).
  opts: {option: value} set for the run.  launches: kernels the call must launch (None: not asserted).  tile: {option:
  value} of the CGAN_OPT_LAST_TC_* geometry the conv kernel launch must report (column tile, tiles per CTA, halo), so
  that a case meant for one kernel instantiation cannot quietly run another."""

  def __init__(self, path, op, n, h, w, cin, cout, kh=1, kw=1, stride=1, up=False, pad="SAME", bias=False,
               residual=False, relu=False, leak=None, opts=None, launches=None, note="", tile=None):
    self.path, self.op, self.n, self.h, self.w, self.cin, self.cout = path, op, n, h, w, cin, cout
    self.kh, self.kw, self.stride, self.up, self.pad = kh, kw, stride, up, pad
    self.bias, self.residual, self.relu, self.leak = bias, residual, relu, leak
    self.opts, self.launches, self.note, self.tile = dict(opts or {}), launches, note, dict(tile or {})

  @property
  def id(self):
    if self.op.startswith("bmm"):
      return "%s-b%d-m%d-n%d-k%d" % (self.op, self.n, self.h, self.w, self.cin)
    s = "%s-n%d-%dx%d-%d-%d-k%dx%d-s%d%s-%s" % (self.op, self.n, self.h, self.w, self.cin, self.cout, self.kh, self.kw,
                                               self.stride, "-up" if self.up else "", self.pad)
    for flag in ("bias", "residual", "relu"):
      if getattr(self, flag):
        s += "-" + flag
    if self.leak is not None:
      s += "-mask%g" % self.leak
    if self.opts.get(_lib.OPT_TC_HALO) == 2:
      s += "-halo"
    return s + ("-" + self.note if self.note else "")


def mt2_batch(sms):
  """A batch for which the per-tap kernel takes two pixel tiles per CTA and the last CTA gets one: on 8x8 maps a tile is
  two images (tc_geometry), tiles_total = ceil(n / 2) must reach 4 x SMs (cgan_conv_tc's rule for mt = 2 at one column
  tile) and be odd.  n itself is odd too, so the last tile also hangs over the batch."""
  tiles = 4 * sms + 1
  return 2 * tiles - 1


def fwd(path, *a, **k):
  return Case(path, "fwd", *a, **k)


def dgrad(path, *a, **k):
  return Case(path, "dgrad", *a, **k)


def wgrad(path, *a, **k):
  return Case(path, "wgrad", *a, **k)


HALO = {_lib.OPT_TC_HALO: 2}
NO_HALO = {_lib.OPT_TC_HALO: 0}
RAN_HALO = {_lib.OPT_LAST_TC_HALO: 1}


def bn(width, mt=1):
  """The launch geometry of a per-tap kernel with `width`-wide column tiles and `mt` pixel tiles per CTA."""
  return {_lib.OPT_LAST_TC_BN: width, _lib.OPT_LAST_TC_MT: mt, _lib.OPT_LAST_TC_HALO: 0}


FWD_CASES = [
    # dense stride 1, even and odd kernels (k = 2 and 4 pad asymmetrically), rectangular maps
    fwd("fwd per-tap", 2, 11, 20, 32, 64, 2, 2, bias=True, launches=2),
    fwd("fwd per-tap", 2, 9, 16, 64, 96, 3, 3, bias=True, residual=True, relu=True, opts=NO_HALO, launches=2),
    fwd("fwd per-tap", 2, 11, 20, 32, 64, 4, 4, bias=True, launches=2),
    fwd("fwd per-tap", 2, 9, 16, 32, 48, 5, 5, residual=True, launches=2),
    # Inception's factorised kernels, square 17x17 and rectangular
    fwd("fwd per-tap", 2, 17, 17, 64, 64, 1, 7, bias=True, launches=2),
    fwd("fwd per-tap", 2, 17, 17, 64, 64, 7, 1, bias=True, launches=2),
    fwd("fwd per-tap", 2, 17, 17, 32, 64, 1, 3, bias=True, launches=2),
    fwd("fwd per-tap", 2, 17, 17, 32, 64, 3, 1, bias=True, launches=2),
    fwd("fwd per-tap", 2, 10, 23, 64, 32, 1, 7, bias=True, launches=2),
    fwd("fwd per-tap", 2, 23, 10, 64, 32, 7, 1, bias=True, launches=2),
    fwd("fwd per-tap", 2, 12, 19, 32, 64, 1, 3, launches=2),
    fwd("fwd per-tap", 2, 19, 12, 32, 64, 3, 1, launches=2),
    # VALID stride 1
    fwd("fwd per-tap", 2, 13, 18, 32, 64, 3, 3, pad="VALID", bias=True, launches=2),
    fwd("fwd per-tap", 2, 12, 9, 32, 32, 4, 2, pad="VALID", launches=2),
    # rows wider than one 128-pixel box
    fwd("fwd per-tap", 1, 3, 129, 32, 32, 3, 3, bias=True, opts=NO_HALO, launches=2),
    fwd("fwd per-tap", 1, 2, 147, 32, 64, 3, 3, opts=NO_HALO, launches=2),
    fwd("fwd per-tap", 1, 2, 257, 32, 32, 3, 3, bias=True, opts=NO_HALO, launches=2),
    # K not a multiple of 32 (zero-padded channel chunk)
    fwd("fwd per-tap", 2, 8, 12, 12, 32, 3, 3, bias=True, opts=NO_HALO, launches=2),
    fwd("fwd per-tap", 2, 9, 10, 20, 32, 3, 3, opts=NO_HALO, launches=2),
    fwd("fwd per-tap", 2, 7, 12, 40, 64, 3, 3, bias=True, opts=NO_HALO, launches=2),
    # odd column counts: the element-by-element epilogue (vec2 = 0)
    fwd("fwd per-tap", 2, 8, 10, 32, 5, 3, 3, bias=True, residual=True, relu=True, opts=NO_HALO, launches=2),
    fwd("fwd per-tap", 2, 8, 10, 32, 33, 3, 3, bias=True, residual=True, opts=NO_HALO, launches=2),
    fwd("fwd per-tap", 2, 9, 7, 32, 75, 3, 3, bias=True, relu=True, opts=NO_HALO, launches=2),
    # > 256 columns, several column tiles: 288 -> 3 x 96; with only two pixel tiles the occupancy rule of
    # tc_pick_bn_occupancy narrows 320 to 5 x 64 (2 x 160 when the grid fills the SMs: wide_cases)
    fwd("fwd per-tap", 2, 8, 16, 32, 288, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=bn(96)),
    fwd("fwd per-tap", 2, 8, 16, 32, 320, 3, 3, bias=True, residual=True, opts=NO_HALO, launches=2, tile=bn(64)),
    # column tiles no occupancy rule narrows: 160 (no divisor in [64, 160)) and 200 -> one 224-wide tile, columns masked
    fwd("fwd per-tap", 2, 8, 16, 32, 160, 3, 3, bias=True, relu=True, opts=NO_HALO, launches=2, tile=bn(160)),
    fwd("fwd per-tap", 2, 9, 14, 32, 200, 3, 3, bias=True, residual=True, opts=NO_HALO, launches=2, tile=bn(224)),
    # sub-pixel phases over a zero-inserted input (k = 5: phases of 9, 6, 6 and 4 taps)
    fwd("fwd phases", 2, 6, 9, 32, 64, 3, 3, up=True, bias=True, launches=2),
    fwd("fwd phases", 2, 6, 9, 32, 64, 4, 4, up=True, bias=True, residual=True, launches=2),
    fwd("fwd phases", 2, 5, 7, 32, 32, 5, 5, up=True, bias=True, relu=True, launches=2),
    # 1x1 over a zero-inserted input: phase 0 on the tensor cores, the bias-only phases, the post pass
    fwd("fwd 1x1-up", 2, 8, 6, 64, 32, 1, 1, up=True, bias=True, launches=3),
    fwd("fwd 1x1-up", 2, 5, 7, 32, 64, 1, 1, up=True, bias=True, residual=True, relu=True, launches=4),
    # stride 2 through the four parity views: SAME and VALID, even and odd extents
    fwd("fwd s2 views", 2, 16, 12, 32, 64, 4, 4, stride=2, bias=True, launches=2),
    fwd("fwd s2 views", 2, 15, 11, 32, 64, 3, 3, stride=2, bias=True, residual=True, launches=2),
    fwd("fwd s2 views", 2, 17, 14, 32, 48, 3, 3, stride=2, pad="VALID", bias=True, launches=2),
    fwd("fwd s2 views", 2, 12, 9, 32, 64, 4, 4, stride=2, pad="VALID", relu=True, launches=2),
    fwd("fwd s2 views", 2, 13, 10, 32, 64, 4, 3, stride=2, launches=2),
    # the halo kernel (three taps of a kernel column share one box), forced
    fwd("fwd halo", 2, 8, 32, 32, 64, 3, 3, bias=True, residual=True, opts=HALO, launches=2, tile=RAN_HALO),
    fwd("fwd halo", 2, 16, 16, 64, 64, 3, 3, bias=True, relu=True, opts=HALO, launches=2, tile=RAN_HALO),
    fwd("fwd halo", 2, 12, 32, 32, 33, 3, 3, bias=True, opts=HALO, launches=2, tile=RAN_HALO),
    # image-side layers: cin <= 4 (patch gather + one GEMM) and cout <= 4 (one GEMM + shift-add)
    fwd("fwd thin-cin", 2, 12, 20, 3, 32, 3, 3, bias=True),
    fwd("fwd thin-cin", 2, 10, 14, 1, 64, 5, 5, bias=True, relu=True),
    fwd("fwd thin-cin", 2, 9, 16, 4, 16, 1, 7, bias=True),
    fwd("fwd thin-cin", 2, 33, 29, 3, 32, 3, 3, stride=2, pad="VALID", bias=True),
    fwd("fwd thin-cout", 2, 12, 20, 64, 3, 3, 3, bias=True),
    fwd("fwd thin-cout", 2, 10, 12, 32, 1, 5, 5, bias=True, relu=True),
    fwd("fwd thin-cout", 2, 9, 14, 32, 4, 1, 7, bias=True, residual=True),
]

DGRAD_CASES = [
    dgrad("dgrad per-tap", 2, 9, 14, 48, 64, 3, 3, launches=2),
    dgrad("dgrad per-tap", 2, 11, 10, 32, 64, 4, 4, bias=True, launches=2),
    dgrad("dgrad per-tap", 2, 10, 17, 64, 32, 1, 7, launches=2),
    dgrad("dgrad per-tap", 2, 8, 12, 5, 64, 3, 3, bias=True, launches=2),
    dgrad("dgrad per-tap", 2, 8, 12, 33, 64, 3, 3, bias=True, leak=0.2, launches=2),
    dgrad("dgrad per-tap", 2, 9, 14, 48, 64, 3, 3, bias=True, leak=0.0, launches=2),
    dgrad("dgrad per-tap", 2, 8, 16, 160, 32, 3, 3, bias=True, leak=0.2, launches=2, tile=bn(160)),
    dgrad("dgrad per-tap", 2, 9, 14, 200, 32, 3, 3, bias=True, launches=2, tile=bn(224)),
    dgrad("dgrad phases", 2, 5, 7, 32, 64, 3, 3, up=True, bias=True, launches=2),
    dgrad("dgrad phases", 2, 5, 7, 64, 32, 4, 4, up=True, leak=0.2, launches=2),
    dgrad("dgrad s2 phases", 2, 12, 16, 32, 64, 4, 4, stride=2, bias=True, launches=2),
    dgrad("dgrad s2 phases", 2, 14, 10, 64, 32, 3, 3, stride=2, leak=0.0, launches=2),
    dgrad("dgrad thin-cout", 2, 12, 20, 64, 3, 3, 3, bias=True),
    dgrad("dgrad thin-cout", 2, 10, 12, 32, 1, 5, 5),
    dgrad("dgrad thin-cin", 2, 12, 20, 3, 32, 3, 3, bias=True),
    dgrad("dgrad thin-cin", 2, 9, 16, 4, 16, 1, 7, leak=0.2),
]

WGRAD_CASES = [
    wgrad("wgrad", 2, 16, 8, 64, 64, 3, 3),
    wgrad("wgrad", 1, 8, 8, 64, 64, 3, 3, launches=1, note="one-split"),
    wgrad("wgrad", 32, 16, 16, 64, 64, 3, 3, launches=2, note="split-k"),
    wgrad("wgrad", 2, 8, 16, 96, 64, 3, 3),
    wgrad("wgrad", 2, 8, 8, 160, 64, 3, 3),
    wgrad("wgrad", 2, 8, 16, 64, 20, 3, 3),
    wgrad("wgrad", 2, 8, 16, 64, 384, 3, 3),
    wgrad("wgrad", 2, 8, 16, 64, 64, 1, 7),
    wgrad("wgrad", 2, 16, 8, 64, 64, 4, 4),
    wgrad("wgrad up", 2, 8, 4, 64, 64, 3, 3, up=True),
    wgrad("wgrad up", 2, 4, 8, 64, 32, 4, 4, up=True),
    wgrad("wgrad s2", 2, 16, 32, 64, 64, 4, 4, stride=2),
    wgrad("wgrad s2", 2, 16, 8, 96, 32, 3, 3, stride=2),
    wgrad("wgrad thin-cin", 2, 16, 16, 3, 32, 3, 3),
    wgrad("wgrad thin-cin", 2, 8, 16, 1, 64, 5, 5),
    wgrad("wgrad thin-cout", 2, 16, 16, 64, 3, 3, 3),
    wgrad("wgrad thin-cout", 2, 8, 16, 128, 1, 5, 5),
]

BMM_CASES = [
    # op, batch, m, n, k (a [b, m, k] / [b, k, m] for tn; rows as an h x w grid: 384 = 3 x 128, 640 = 5 x 128)
    Case("bmm nt/nn", "bmm_nt", 3, 384, 40, 24, 0, launches=2),
    Case("bmm nt/nn", "bmm_nn", 3, 640, 36, 16, 0, launches=2),
    Case("bmm nt/nn", "bmm_nt", 2, 128, 100, 8, 0, launches=2),
    Case("bmm tn", "bmm_tn", 3, 64, 20, 256, 0, launches=1),
    Case("bmm tn", "bmm_tn", 2, 96, 256, 384, 0, launches=1),
]

ALL_CASES = FWD_CASES + DGRAD_CASES + WGRAD_CASES + BMM_CASES


def wide_cases(sms):
  """Column tiles of 128, 160, 192 and 256 (the 128 / 256-channel layers of the GANs, Inception's 160 / 192 / 320): the
  occupancy rule (tc_pick_bn_occupancy) keeps a tile this wide only when there are enough pixel tiles to fill the SMs,
  so the batches are sized from the SM count.  On 8x16 maps a pixel tile is one image; an image of the 384-row batched
  GEMM is three; a 32-wide halo tile covers four rows of 8x32, so two per image."""
  full, half, third = sms, -(-sms // 2), -(-sms // 3)
  return [
      fwd("fwd per-tap", half, 8, 16, 16, 320, 3, 3, bias=True, residual=True, opts=NO_HALO, launches=2, tile=bn(160)),
      fwd("fwd per-tap", full, 8, 16, 16, 256, 3, 3, bias=True, relu=True, opts=NO_HALO, launches=2, tile=bn(256)),
      fwd("fwd per-tap", full, 8, 16, 16, 192, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=bn(192)),
      fwd("fwd per-tap", full, 8, 16, 16, 128, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=bn(128)),
      fwd("fwd halo", half, 8, 32, 16, 256, 3, 3, bias=True, opts=HALO, launches=2, tile={**bn(256), **RAN_HALO}),
      # (a 256-column dgrad whose operand is rounded in the kernel would take the halo kernel by default)
      dgrad("dgrad per-tap", full, 8, 16, 256, 16, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=bn(256)),
      dgrad("dgrad per-tap", full, 8, 16, 192, 16, 3, 3, leak=0.2, opts=NO_HALO, launches=2, tile=bn(192)),
      dgrad("dgrad per-tap", full, 8, 16, 128, 16, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=bn(128)),
      dgrad("dgrad halo", full, 8, 16, 256, 16, 3, 3, bias=True, leak=0.0, launches=2, tile={**bn(256), **RAN_HALO}),
      Case("bmm nt/nn", "bmm_nt", third, 384, 128, 24, 0, launches=2, tile=bn(128)),
      Case("bmm nt/nn", "bmm_nn", third, 384, 256, 16, 0, launches=2, tile=bn(256)),
  ]


# ---------------------------------------------------------------------------------------------------- float64 reference

def tf_pad(size, k, stride, padding):
  """(output extent, padding before, padding after) of one dimension: TF SAME or VALID, from its definition."""
  if padding == "SAME":
    out = -(-size // stride)
    total = max((out - 1) * stride + k - size, 0)
    return out, total // 2, total - total // 2
  return (size - k) // stride + 1, 0, 0


def out_hw(c):
  vh, vw = (2 * c.h, 2 * c.w) if c.up else (c.h, c.w)
  return tf_pad(vh, c.kh, c.stride, c.pad)[0], tf_pad(vw, c.kw, c.stride, c.pad)[0]


def conv64(c, x, w):
  """y[n, oh, ow, co] = sum x_virtual[n, oh * s + kh - pad_t, ow * s + kw - pad_l, ci] * w[kh, kw, ci, co] in float64;
  x is the real NHWC input (zero-inserted to 2h x 2w when c.up), w is HWIO."""
  xt = x.permute(0, 3, 1, 2)
  if c.up:
    z = xt.new_zeros(xt.shape[0], xt.shape[1], 2 * xt.shape[2], 2 * xt.shape[3])
    z[:, :, ::2, ::2] = xt
    xt = z
  oh, pt, pb = tf_pad(xt.shape[2], c.kh, c.stride, c.pad)
  ow, pl, pr = tf_pad(xt.shape[3], c.kw, c.stride, c.pad)
  y = F.conv2d(F.pad(xt, (pl, pr, pt, pb)).contiguous(), w.permute(3, 2, 0, 1).contiguous(), stride=c.stride)
  assert tuple(y.shape[2:]) == (oh, ow), (tuple(y.shape), oh, ow)
  return y.permute(0, 2, 3, 1)


def contract64(c, a, b):
  """The case's contraction of the float32 operands a, b in float64 (CPU).  The input and filter gradients are the
  adjoints of conv64 (torch's conv_transpose2d / conv2d_weight, reached through autograd)."""
  a = torch.from_numpy(np.asarray(a, np.float64))
  b = torch.from_numpy(np.asarray(b, np.float64))
  if c.op == "fwd":
    return conv64(c, a, b).numpy()
  if c.op == "dgrad":
    x = torch.zeros(c.n, c.h, c.w, c.cin, dtype=torch.float64, requires_grad=True)
    return torch.autograd.grad(conv64(c, x, b), x, a)[0].numpy()
  if c.op == "wgrad":
    w = torch.zeros(c.kh, c.kw, c.cin, c.cout, dtype=torch.float64, requires_grad=True)
    return torch.autograd.grad(conv64(c, a, w), w, b)[0].numpy()
  if c.op == "bmm_nt":
    return torch.bmm(a, b.transpose(1, 2)).numpy()
  if c.op == "bmm_nn":
    return torch.bmm(a, b).numpy()
  return torch.bmm(a.transpose(1, 2), b).numpy()         # bmm_tn


def operand_shapes(c):
  if c.op.startswith("bmm"):
    bsz, m, n, k = c.n, c.h, c.w, c.cin
    return {"bmm_nt": ((bsz, m, k), (bsz, n, k)), "bmm_nn": ((bsz, m, k), (bsz, k, n)),
            "bmm_tn": ((bsz, k, m), (bsz, k, n))}[c.op]
  oh, ow = out_hw(c)
  x, dy, w = (c.n, c.h, c.w, c.cin), (c.n, oh, ow, c.cout), (c.kh, c.kw, c.cin, c.cout)
  return {"fwd": (x, w), "dgrad": (dy, w), "wgrad": (x, dy)}[c.op]


def out_shape(c):
  if c.op.startswith("bmm"):
    return (c.n, c.h, c.w)
  oh, ow = out_hw(c)
  return {"fwd": (c.n, oh, ow, c.cout), "dgrad": (c.n, c.h, c.w, c.cin), "wgrad": (c.kh, c.kw, c.cin, c.cout)}[c.op]


def seed_of(c, salt=0):
  return (sum(ord(ch) * (i + 1) for i, ch in enumerate(c.id)) + salt) % (2 ** 31)


def draw(c, salt=0, mask_zeros=True):
  """Seeded TF32-exact operands a, b and the epilogue tensors of the case.  The (leaky-)ReLU mask holds exact +-0 where
  the two rules part ways; mask_zeros=False draws it as it was drawn before it had them (the same normal values)."""
  rng = np.random.RandomState(seed_of(c, salt))
  sa, sb = operand_shapes(c)
  a = rna_tf32(rng.standard_normal(sa).astype(np.float32))
  b = rna_tf32(rng.standard_normal(sb).astype(np.float32))
  shape = out_shape(c)
  ncols = shape[-1]
  ex = {}
  if c.bias:
    ex["bias"] = (4.0 * rng.standard_normal(ncols)).astype(np.float32)
  if c.residual:
    ex["residual"] = (4.0 * rng.standard_normal(shape)).astype(np.float32)
  if c.leak is not None:
    ex["mask"] = relu_mask(rng, shape) if mask_zeros else rng.standard_normal(shape).astype(np.float32)
  return a, b, ex


def reference(c, a, b, ex):
  """(y64, A): the float64 result with the case's epilogue, and the scale of the criterion."""
  y = contract64(c, a, b)
  scale = contract64(c, np.abs(a), np.abs(b))
  if "bias" in ex:
    y = y + ex["bias"].astype(np.float64)
    scale = scale + np.abs(ex["bias"].astype(np.float64))
  if "residual" in ex:
    y = y + ex["residual"]
    scale = scale + np.abs(ex["residual"].astype(np.float64))
  if c.relu:
    y = np.maximum(y, 0.0)
  if "mask" in ex:
    y = relu_gate(ex["mask"], y, c.leak)
  return y, scale


def check(y, y64, scale, what, path=None):
  """The element-wise criterion; returns the worst err / A (and records it per path)."""
  y = np.asarray(y)
  assert y.shape == y64.shape, "%s: shape %s vs %s" % (what, y.shape, y64.shape)
  assert np.isfinite(y).all(), "%s: non-finite values" % what
  err = np.abs(y.astype(np.float64) - y64)
  bad = err > TAU * scale + 1e-30
  ratio = err / np.maximum(scale, 1e-300)
  worst = float(ratio.max()) if ratio.size else 0.0
  if path is not None and worst >= WORST.get(path, (-1.0, ""))[0]:
    WORST[path] = (worst, what)
  if bad.any():
    i = np.unravel_index(int(np.argmax(np.where(bad, ratio, -1.0))), y.shape)
    raise AssertionError("%s: %d of %d elements exceed err <= %.0e * A; worst err/A %.3e at %s (got %.9g, float64 %.9g, A %.4g)"
                         % (what, int(bad.sum()), y.size, TAU, worst, i, float(y[i]), float(y64[i]), float(scale[i])))
  return worst


@pytest.fixture(scope="module", autouse=True)
def _report_worst_ratios(pytestconfig):
  """Prints the worst err / A per path of the library's own results (the emulator run records nothing) to the terminal,
  past pytest's output capture."""
  t0 = time.time()
  WORST.clear()
  yield
  if WORST:
    lines = ["worst err/A per tensor-core path (TAU = %.0e), %.1f s:" % (TAU, time.time() - t0)]
    lines += ["  %-19s %.3e  (%s)" % (path, WORST[path][0], WORST[path][1]) for path in sorted(WORST)]
    capman = pytestconfig.pluginmanager.getplugin("capturemanager")
    tr = pytestconfig.pluginmanager.getplugin("terminalreporter")
    if capman is None or tr is None:
      print("\n".join(lines))
      return
    with capman.global_and_fixture_disabled():       # what capsys.disabled() does
      tr.ensure_newline()
      for line in lines:
        tr.write_line(line)


# ---------------------------------------------------------------------------------------------------- engine side

def emulated(K):
  return bool(getattr(K.lib(), "emulated", False))


class options(object):
  """Sets context options for a block and restores the previous values."""

  def __init__(self, K, opts):
    self.lib, self.opts = K.lib(), dict(opts)

  def __enter__(self):
    self.saved = {k: self.lib.get_option(k) for k in self.opts}
    for k, v in self.opts.items():
      self.lib.set_option(k, v)

  def __exit__(self, *exc):
    for k, v in self.saved.items():
      self.lib.set_option(k, v)


def desc(K, c):
  return K.conv_desc(c.n, c.h, c.w, c.cin, c.cout, c.kh, c.kw, c.stride, c.up, c.pad)


def run(K, c, a, b, ex, round_out=False, in_tf32=False, wflags=0, out=None):
  """One call of the library entry point of the case; returns (result, kernels launched, path taken)."""
  lib = K.lib()
  A, B = K.from_numpy(a), K.from_numpy(b)
  dev = {k: K.from_numpy(v) for k, v in ex.items()}
  y = K.empty(*out_shape(c)) if out is None else out
  n0 = lib.launch_count()
  with options(K, c.opts):
    if c.op.startswith("bmm"):
      y = K.bmm(A, B, ta=c.op == "bmm_tn", tb=c.op == "bmm_nt")
    elif c.op == "wgrad":
      K._call("conv2d_wgrad_ex", ctypes.byref(desc(K, c)), A.ptr, B.ptr, int(wflags), y.ptr)
    else:
      ep = K._epilogue(dev.get("bias"), dev.get("residual"), dev.get("mask"), c.leak or 0.0, c.relu, round_out, in_tf32)
      name = "conv2d_fwd_ex" if c.op == "fwd" else "conv2d_dgrad_ex"
      K._call(name, ctypes.byref(desc(K, c)), A.ptr, B.ptr, ctypes.byref(ep), y.ptr)
  launched = lib.launch_count() - n0
  path = _lib.PATH_NAMES[lib.get_option(_lib.OPT_LAST_PATH)]
  return np.array(y.cpu(), copy=True), launched, path


def assert_path(K, c, launched, path):
  if emulated(K):
    return
  assert path == "tcgen05_tf32", "%s: ran on %s, not the tensor cores" % (c.id, path)
  if c.launches is not None:
    assert launched == c.launches, "%s: %d kernels launched, expected %d" % (c.id, launched, c.launches)
  lib = K.lib()
  got = {key: lib.get_option(key) for key in c.tile}
  assert got == c.tile, "%s: conv kernel launched with %s, expected %s (keys: bn %d, mt %d, halo %d)" % (
      c.id, got, c.tile, _lib.OPT_LAST_TC_BN, _lib.OPT_LAST_TC_MT, _lib.OPT_LAST_TC_HALO)


def same_bits(a, b):
  """Bit-identical float32 arrays (the two zeros count as one: ReLU may return either)."""
  a, b = np.asarray(a, np.float32) + np.float32(0.0), np.asarray(b, np.float32) + np.float32(0.0)
  return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def check_case(K, c, record=True):
  a, b, ex = draw(c)
  y64, scale = reference(c, a, b, ex)
  first, launched, path = run(K, c, a, b, ex)
  assert_path(K, c, launched, path)
  second = run(K, c, a, b, ex)[0]
  assert np.array_equal(first.view(np.uint32), second.view(np.uint32)), "%s: two runs differ" % c.id
  return check(first, y64, scale, c.id, c.path if record else None)


@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  kernels.set_math_mode(1)
  yield kernels
  kernels.set_math_mode(0)


# ---------------------------------------------------------------------------------------------------- element-wise cases

@pytest.mark.gpu
@pytest.mark.parametrize("c", ALL_CASES, ids=[c.id for c in ALL_CASES])
def test_tc_contraction_elementwise(K, c):
  check_case(K, c)


WIDE_IDS = [c.id.replace("-n%d-" % c.n, "-nSM-").replace("-b%d-" % c.n, "-bSM-") for c in wide_cases(132)]


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(WIDE_IDS)), ids=WIDE_IDS)
def test_wide_column_tiles_elementwise(K, i):
  """The 128- to 256-wide column tiles, at batches (from the SM count) large enough that the occupancy rule keeps them;
  each case asserts the tile width its launch reported."""
  check_case(K, wide_cases(torch.cuda.get_device_properties(0).multi_processor_count)[i])


def mt2_cases(sms):
  n = mt2_batch(sms)
  return [fwd("fwd per-tap", n, 8, 8, 32, 64, 3, 3, bias=True, opts=NO_HALO, launches=2, note="mt2-odd",
              tile=bn(64, mt=2)),
          dgrad("dgrad per-tap", n, 8, 8, 32, 64, 3, 3, bias=True, opts=NO_HALO, launches=2, note="mt2-odd",
                tile=bn(32, mt=2))]


def tiles_total_8x8(n):
  return (n + 1) // 2


@pytest.mark.gpu
def test_two_tiles_per_cta_with_an_odd_tile_count(K):
  """mt = 2 and an odd number of pixel tiles (the last CTA multiplies a stale second tile and stores only its first):
  element-wise exact, and bit-identical to mt = 1, for the forward and the input gradient."""
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  for c in mt2_cases(sms):
    tiles = tiles_total_8x8(c.n)
    assert tiles % 2 == 1 and tiles >= 4 * sms
    check_case(K, c)
    a, b, ex = draw(c)
    mt2 = run(K, c, a, b, ex)[0]
    with options(K, {_lib.OPT_TC_MT: 1}):
      mt1 = run(K, c, a, b, ex)[0]
      assert K.lib().get_option(_lib.OPT_LAST_TC_MT) == 1
    assert same_bits(mt2, mt1), "%s: mt = 2 and mt = 1 differ" % c.id


@pytest.mark.gpu
@pytest.mark.parametrize("kh,kw,stride,pad", [(3, 3, 1, "SAME"), (1, 7, 1, "SAME"), (3, 3, 2, "VALID"), (4, 4, 2, "SAME")])
def test_channel_slice_output(K, kh, kw, stride, pad):
  """A forward convolution stored into channels [24, 24 + cout) of a wider NHWC tensor (ChannelSink): element-wise
  exact, bit-identical to the dense output, and the neighbouring channels keep their bits."""
  check_channel_slice(K, kh, kw, stride, pad)


def check_channel_slice(K, kh, kw, stride, pad, record=True):
  c = fwd("fwd sliced", 2, 13, 10, 32, 36, kh, kw, stride=stride, pad=pad, bias=True, relu=True, opts=NO_HALO, launches=2)
  a, b, ex = draw(c)
  y64, scale = reference(c, a, b, ex)
  oh, ow = out_hw(c)
  sink = K.ChannelSink(c.cout + 40)
  buf = sink.buffer(c.n, oh, ow)
  fill = np.random.RandomState(1).standard_normal((c.n, oh, ow, c.cout + 40)).astype(np.float32)
  K.copy_(buf, K.from_numpy(fill))
  dense, _, _ = run(K, c, a, b, ex)
  lib = K.lib()
  A, B, bias = K.from_numpy(a), K.from_numpy(b), K.from_numpy(ex["bias"])
  n0 = lib.launch_count()
  with options(K, c.opts):
    ep = K._epilogue(bias, relu=True, ldy=sink.channels)
    K._call("conv2d_fwd_ex", ctypes.byref(desc(K, c)), A.ptr, B.ptr, ctypes.byref(ep), buf.ptr + 4 * 24)
  assert_path(K, c, lib.launch_count() - n0, _lib.PATH_NAMES[lib.get_option(_lib.OPT_LAST_PATH)])
  got = np.array(buf.cpu(), copy=True)
  check(got[..., 24:24 + c.cout], y64, scale, c.id + "-slice", c.path if record else None)
  assert same_bits(got[..., 24:24 + c.cout], dense), "sliced and dense outputs differ"
  assert np.array_equal(got[..., :24].view(np.uint32), fill[..., :24].view(np.uint32))
  assert np.array_equal(got[..., 24 + c.cout:].view(np.uint32), fill[..., 24 + c.cout:].view(np.uint32))


# ---------------------------------------------------------------------------------------------------- bit-exact invariants

EPILOGUE_CASES = [
    fwd("fwd per-tap", 2, 9, 16, 64, 96, 3, 3, opts=NO_HALO),
    fwd("fwd per-tap", 2, 8, 10, 32, 33, 3, 3, opts=NO_HALO),
    fwd("fwd halo", 2, 8, 32, 32, 64, 3, 3, opts=HALO),
    fwd("fwd phases", 2, 6, 9, 32, 64, 4, 4, up=True),
    fwd("fwd s2 views", 2, 15, 11, 32, 64, 3, 3, stride=2),
    fwd("fwd 1x1-up", 2, 5, 7, 32, 64, 1, 1, up=True),
    dgrad("dgrad per-tap", 2, 8, 12, 33, 64, 3, 3),
    dgrad("dgrad phases", 2, 5, 7, 64, 32, 4, 4, up=True),
    dgrad("dgrad s2 phases", 2, 12, 16, 32, 64, 4, 4, stride=2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("c", EPILOGUE_CASES, ids=[c.id for c in EPILOGUE_CASES])
def test_fused_epilogue_is_exact_fp32_algebra(K, c):
  """On the wgmma conv kernels the epilogue acts on the accumulator y0 in a fixed order: + bias, + residual, ReLU,
  the (leaky-)ReLU gate, TF32 rounding.  Each fused result equals that algebra applied in fp32 to y0 (the same kernel
  without any epilogue), bit for bit."""
  rng = np.random.RandomState(seed_of(c, 7))
  a, b, _ = draw(c)
  shape = out_shape(c)
  bias = (4.0 * rng.standard_normal(shape[-1])).astype(np.float32)
  res = (4.0 * rng.standard_normal(shape)).astype(np.float32)
  mask = relu_mask(rng, shape)
  f = np.float32

  def with_ep(round_out=False, **ep):
    cc = Case(c.path, c.op, c.n, c.h, c.w, c.cin, c.cout, c.kh, c.kw, c.stride, c.up, c.pad, opts=c.opts,
              bias="bias" in ep, residual="residual" in ep, relu=ep.get("relu", False), leak=ep.get("leak"))
    ex = {k: v for k, v in (("bias", bias), ("residual", res), ("mask", mask)) if k in ep or (k == "mask" and "leak" in ep)}
    y, launched, path = run(K, cc, a, b, ex, round_out=round_out)
    assert_path(K, cc, launched, path)
    return y

  y0 = with_ep()
  yb = (y0 + bias).astype(f)
  assert same_bits(with_ep(bias=1), yb), "%s: + bias" % c.id
  assert same_bits(with_ep(leak=0.2), relu_gate(mask, y0, 0.2)), "%s: mask without bias" % c.id
  for leak in (0.0, 0.2):
    assert same_bits(with_ep(bias=1, leak=leak), relu_gate(mask, yb, leak)), "%s: + bias, mask %g" % (c.id, leak)
  assert same_bits(with_ep(round_out=True, bias=1), rna_tf32(yb)), "%s: + bias, rounded" % c.id
  if c.op == "fwd":           # the forward entry takes the residual and the plain ReLU as well
    ybr = (yb + res).astype(f)
    assert same_bits(with_ep(bias=1, residual=1), ybr), "%s: + bias + residual" % c.id
    ybrr = np.maximum(ybr, f(0))
    assert same_bits(with_ep(bias=1, residual=1, relu=True), ybrr), "%s: + bias + residual, ReLU" % c.id
    assert same_bits(with_ep(round_out=True, bias=1, residual=1, relu=True), rna_tf32(ybrr)), "%s: all, rounded" % c.id


PRE_ROUNDED_CASES = [
    fwd("fwd per-tap", 2, 9, 16, 64, 96, 3, 3),
    fwd("fwd phases", 2, 6, 9, 32, 64, 3, 3, up=True),
    fwd("fwd s2 views", 2, 16, 12, 32, 64, 4, 4, stride=2),
    fwd("fwd thin-cout", 2, 12, 20, 64, 3, 3, 3),
    dgrad("dgrad per-tap", 2, 9, 14, 48, 64, 3, 3),
    dgrad("dgrad phases", 2, 5, 7, 32, 64, 3, 3, up=True),
    dgrad("dgrad s2 phases", 2, 12, 16, 32, 64, 4, 4, stride=2),
    dgrad("dgrad thin-cin", 2, 12, 20, 3, 32, 3, 3),
    wgrad("wgrad", 2, 16, 8, 64, 64, 3, 3),
    wgrad("wgrad up", 2, 8, 4, 64, 64, 3, 3, up=True),
    wgrad("wgrad s2", 2, 16, 32, 64, 64, 4, 4, stride=2),
    wgrad("wgrad thin-cin", 2, 16, 16, 3, 32, 3, 3),
    wgrad("wgrad thin-cout", 2, 16, 16, 64, 3, 3, 3),
]


@pytest.mark.gpu
@pytest.mark.parametrize("c", PRE_ROUNDED_CASES, ids=[c.id for c in PRE_ROUNDED_CASES])
def test_pre_rounded_flags_change_no_bit(K, c):
  """CGAN_CONV_IN_TF32 / IN2_TF32 only skip the rounding of operands that are already TF32 values: on such operands the
  results with the flags set and cleared are bit-identical.  The halo kernel is pinned off, because the flag also
  decides whether the halo kernel is used."""
  a, b, ex = draw(c)
  opts = dict(c.opts)
  opts[_lib.OPT_TC_HALO] = 0
  cc = Case(c.path, c.op, c.n, c.h, c.w, c.cin, c.cout, c.kh, c.kw, c.stride, c.up, c.pad, opts=opts)
  plain, l0, p0 = run(K, cc, a, b, ex)
  flagged, l1, p1 = run(K, cc, a, b, ex, in_tf32=True, wflags=_lib.CONV_IN_TF32 | _lib.CONV_IN2_TF32)
  assert_path(K, cc, l0, p0)
  assert_path(K, cc, l1, p1)
  assert same_bits(plain, flagged), "%s: pre-rounded flags changed the result" % c.id


# ---------------------------------------------------------------------------------------------------- rounding mode

def rounding_probe(rng, shape):
  """Positive fp32 values whose 13 low mantissa bits are an exact TF32 rounding tie (half of them), one unit above a
  tie or one unit below.  The kept mantissa is even, so round-to-nearest-even takes every tie DOWN where cvt.rna takes
  it up, and truncation takes ties and the values above them down: either moves err / A by several 1e-4."""
  base = rng.uniform(0.5, 2.0, shape).astype(np.float32).view(np.uint32) & np.uint32(0xFFFFC000)
  low = rng.choice(np.array([0x1000, 0x1000, 0x1001, 0x0FFF], np.uint32), size=shape)
  return (base | low).view(np.float32)


def rne_tf32(a):
  u = np.ascontiguousarray(a, np.float32).view(np.uint32)
  return ((u + np.uint32(0xFFF) + ((u >> np.uint32(13)) & np.uint32(1))) & np.uint32(0xFFFFE000)).view(np.float32)


def trunc_tf32(a):
  return (np.ascontiguousarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


ROUNDING_CASES = [
    # (case, probe a, probe b): which operands carry unrounded values (the others are TF32-exact)
    (fwd("fwd per-tap", 2, 9, 16, 64, 96, 3, 3, opts=NO_HALO, note="smem-rounding"), True, False),
    (fwd("fwd per-tap", 2, 9, 16, 64, 96, 3, 3, opts=NO_HALO, note="wprep"), False, True),
    (fwd("fwd halo", 2, 8, 32, 32, 64, 3, 3, opts=HALO, note="rounding"), True, True),
    (fwd("fwd phases", 2, 6, 9, 32, 64, 4, 4, up=True, note="rounding"), True, True),
    (fwd("fwd s2 views", 2, 15, 11, 32, 64, 3, 3, stride=2, note="rounding"), True, True),
    (dgrad("dgrad per-tap", 2, 9, 14, 48, 64, 3, 3, note="rounding"), True, True),
    (fwd("fwd thin-cin", 2, 12, 20, 3, 32, 3, 3, note="patch-gather"), True, True),
    (fwd("fwd thin-cout", 2, 12, 20, 64, 3, 3, 3, note="rounding"), True, True),
    (dgrad("dgrad thin-cout", 2, 12, 20, 64, 3, 3, 3, note="patch-gather"), True, True),
    (dgrad("dgrad thin-cin", 2, 12, 20, 3, 32, 3, 3, note="rounding"), True, True),
    (wgrad("wgrad", 2, 16, 8, 64, 64, 3, 3, note="transpose-rounding"), True, True),
    (wgrad("wgrad up", 2, 8, 4, 64, 64, 3, 3, up=True, note="transpose-rounding"), True, True),
    (wgrad("wgrad s2", 2, 16, 32, 64, 64, 4, 4, stride=2, note="transpose-rounding"), True, True),
    (wgrad("wgrad thin-cin", 2, 16, 16, 3, 32, 3, 3, note="patch-gather"), True, True),
    (wgrad("wgrad thin-cout", 2, 16, 16, 64, 3, 3, 3, note="patch-gather"), True, True),
    (Case("bmm nt/nn", "bmm_nt", 3, 384, 40, 24, 0, note="rounding"), True, True),
    (Case("bmm tn", "bmm_tn", 3, 64, 20, 256, 0, note="rounding"), True, True),
]


def check_rounding_case(K, c, probe_a, probe_b, record=True):
  a, b, _ = draw(c)
  rng = np.random.RandomState(seed_of(c, 3))
  if probe_a:
    a = rounding_probe(rng, a.shape)
  if probe_b:
    b = rounding_probe(rng, b.shape)
  else:
    b = np.abs(b)
  if not probe_a:
    a = np.abs(a)
  y, launched, path = run(K, c, a, b, {})
  assert_path(K, c, launched, path)
  y64, scale = reference(c, rna_tf32(a), rna_tf32(b), {})
  return check(y, y64, scale, c.id + " (unrounded operands vs float64 on their cvt.rna values)",
               c.path + " rna" if record else None)


@pytest.mark.gpu
@pytest.mark.parametrize("c,probe_a,probe_b", ROUNDING_CASES, ids=[r[0].id for r in ROUNDING_CASES])
def test_operand_rounding_is_round_to_nearest_ties_away(K, c, probe_a, probe_b):
  """Operands that are NOT pre-rounded, all positive, built at TF32 rounding ties and next to them: the result must
  match float64 on the cvt.rna values of the operands element by element.  Each case pins one place where an operand is
  rounded: the conv kernel's shared-memory pass (per-tap and halo), the weight preparation, the thin paths' patch
  gather, the filter-gradient transpose and the batched products."""
  check_rounding_case(K, c, probe_a, probe_b)


# ---------------------------------------------------------------------------------------------------- CPU tests

def test_criterion_accepts_fp32_and_rejects_local_defects():
  """The criterion is neither tighter than fp32 accumulation nor too loose for a local defect: an fp32 CPU evaluation
  of TF32-exact operands passes at K = 4608, and four defects built from the float64 result each fail: one tap dropped
  at one border pixel, one 8-channel k-step dropped for one output column, truncated operands, and operands rounded to
  nearest-even."""
  c = fwd("self-test", 1, 6, 7, 512, 16, 3, 3)
  a, b, _ = draw(c)
  y64, scale = reference(c, a, b, {})
  y32 = conv64(c, torch.from_numpy(a), torch.from_numpy(b)).numpy()          # float32: torch keeps the input dtype
  assert y32.dtype == np.float32
  ok = check(y32, y64, scale, "fp32 CPU evaluation")
  assert ok < TAU / 4, ok

  def rejected(y, what):
    with pytest.raises(AssertionError):
      check(y, y64, scale, what)

  # 1. tap (kh, kw) = (1, 1) missing at the border pixel (0, 0, 3): it reads x[0, 0, 3]
  y = y64.copy()
  y[0, 0, 3] -= a[0, 0, 3].astype(np.float64) @ b[1, 1].astype(np.float64)
  rejected(y, "one tap dropped at one border pixel")
  # 2. channels 8..15 of the centre tap (1, 1) missing for output column 5 (the centre tap reads the output's own pixel)
  y = y64.copy()
  y[..., 5] -= a[..., 8:16].astype(np.float64) @ b[1, 1, 8:16, 5].astype(np.float64)
  rejected(y, "one 8-channel k-step of one tap dropped for one column")
  # 3 / 4. unrounded positive operands at and next to rounding ties, rounded by truncation / to nearest-even
  rng = np.random.RandomState(5)
  pa, pb = rounding_probe(rng, a.shape), rounding_probe(rng, b.shape)
  y64, scale = reference(c, rna_tf32(pa), rna_tf32(pb), {})
  ok = check(conv64(c, torch.from_numpy(rna_tf32(pa)), torch.from_numpy(rna_tf32(pb))).numpy(), y64, scale, "fp32, rna")
  assert ok < TAU / 4, ok
  rejected(contract64(c, trunc_tf32(pa), trunc_tf32(pb)), "truncated operands")
  rejected(contract64(c, rne_tf32(pa), rne_tf32(pb)), "round-to-nearest-even operands")


def test_elementwise_cases_on_the_emulator():
  """The element-wise and rounding cases against tests/abi_emulator.py (fp32 CPU evaluation on cvt.rna-rounded operands):
  shows that the reference, the criterion and the case geometry agree with the C-ABI's contract without a GPU.  The
  assertions on the path taken, the launch count and the launch geometry are specific to the real library and are
  skipped, and the emulator's ratios stay out of the per-path report."""
  from compare_gan_b200 import kernels
  with emulated_library():
    kernels.set_math_mode(1)
    try:
      for c in ALL_CASES + wide_cases(132) + mt2_cases(132):
        check_case(kernels, c, record=False)
      for args in ROUNDING_CASES:
        check_rounding_case(kernels, *args, record=False)
      check_channel_slice(kernels, 3, 3, 1, "SAME", record=False)
    finally:
      kernels.set_math_mode(0)
