"""The residual and ReLU-mask operands that the per-tap wgmma convolution prefetches into its stage ring by TMA
(tile_epilogue_smem in csrc/conv_tc.cu), element by element against float64 by the criterion of test_tc_exact_gpu.py,
where that file's cases do not reach: tiles that hang over the grid (17x17 and 35x35 maps: 119 and 105 of 128 rows),
two pixel tiles per CTA at a 64-wide column tile, the 256-wide tile at one CTA per SM, the 128-wide tile at two, the
output phases of an up-sampling forward and a stride-2 input gradient, the masked input gradient of an up-sampling
convolution (nine taps over four parity views of dy), and an output stored into a channel slice of a wider tensor.

Every case also asserts which epilogue ran (CGAN_OPT_LAST_TC_EP_SMEM) and that the prefetched epilogue is the fp32
algebra of the register epilogue, bit for bit: y0 (the same launch with no epilogue operand, which reads nothing from
global memory) + bias + residual, ReLU, the (leaky-)ReLU gate, TF32 rounding.  Launches the prefetch does not serve
(an odd column count, a residual and a mask together) report the register epilogue."""
import ctypes

import numpy as np
import pytest
import torch

from compare_gan_b200 import _lib
from tests.abi_emulator import relu_gate, rna_tf32
from tests.test_tc_exact_gpu import (K, NO_HALO, Case, assert_path, check, check_case, desc, dgrad, draw, fwd,  # noqa: F401
                                     mt2_batch, options, out_hw, reference, run, same_bits)

EP = _lib.OPT_LAST_TC_EP_SMEM


def tile(width=None, mt=None, ctas=None, ep=1):
  t = {EP: ep, _lib.OPT_LAST_TC_HALO: 0}
  for key, v in ((_lib.OPT_LAST_TC_BN, width), (_lib.OPT_LAST_TC_MT, mt), (_lib.OPT_LAST_TC_CTAS_PER_SM, ctas)):
    if v is not None:
      t[key] = v
  return t


def cases(sms):
  two, mt2 = 2 * sms, mt2_batch(sms)
  return [
      # tiles hanging over the grid: 17x7 and 35x3 boxes, the border rows zero-filled by TMA and never stored
      fwd("fwd per-tap", 2, 17, 17, 32, 64, 3, 3, bias=True, residual=True, opts=NO_HALO, launches=2, tile=tile(64)),
      fwd("fwd per-tap", 2, 35, 35, 32, 64, 3, 3, bias=True, residual=True, relu=True, opts=NO_HALO, launches=2,
          tile=tile(64)),
      dgrad("dgrad per-tap", 2, 17, 17, 64, 64, 3, 3, bias=True, leak=0.0, launches=2, tile=tile(64)),
      dgrad("dgrad per-tap", 2, 35, 35, 64, 32, 3, 3, leak=0.2, launches=2, tile=tile(64)),
      # two pixel tiles per CTA at bn = 64, an odd tile count: the last CTA prefetches for its first tile only
      fwd("fwd per-tap", mt2, 8, 8, 32, 64, 3, 3, bias=True, residual=True, opts=NO_HALO, launches=2, note="mt2-odd",
          tile=tile(64, mt=2, ctas=2)),
      dgrad("dgrad per-tap", mt2, 8, 8, 64, 32, 3, 3, leak=0.0, opts=NO_HALO, launches=2, note="mt2-odd",
            tile=tile(64, mt=2, ctas=2)),
      # 256 columns: the 128-wide tile at two CTAs per SM (G's 256-channel layers), and the 256-wide tile at one
      fwd("fwd per-tap", two, 8, 16, 256, 256, 3, 3, bias=True, residual=True, opts=NO_HALO, launches=2,
          tile=tile(128, mt=1, ctas=2)),
      dgrad("dgrad per-tap", two, 8, 16, 256, 256, 3, 3, bias=True, leak=0.0, opts=NO_HALO, launches=2,
            tile=tile(128, mt=1, ctas=2)),
      fwd("fwd per-tap", two, 8, 16, 352, 256, 3, 3, bias=True, residual=True, opts=NO_HALO, launches=2, note="long-k",
          tile=tile(256, mt=1, ctas=1)),
      dgrad("dgrad per-tap", two - 1, 8, 16, 256, 128, 3, 3, leak=0.0, opts=NO_HALO, launches=2, note="below-2-waves",
            tile=tile(256, mt=1, ctas=1)),
      # phases: the forward of an up-sampling convolution writes four output phases (one residual view per phase), its
      # input gradient reads dy through four parity views, a stride-2 input gradient writes four output phases
      fwd("fwd phases", 2, 6, 9, 32, 64, 4, 4, up=True, bias=True, residual=True, launches=2, tile=tile(64)),
      fwd("fwd phases", 2, 5, 7, 32, 96, 3, 3, up=True, residual=True, relu=True, launches=2, tile=tile(96)),
      dgrad("dgrad phases", 2, 5, 7, 64, 32, 3, 3, up=True, leak=0.0, launches=2, tile=tile(64)),
      dgrad("dgrad phases", 2, 8, 8, 128, 64, 4, 4, up=True, bias=True, leak=0.2, launches=2, tile=tile(64)),
      dgrad("dgrad s2 phases", 2, 14, 10, 64, 32, 3, 3, stride=2, leak=0.0, launches=2, tile=tile(64)),
      dgrad("dgrad s2 phases", 2, 12, 16, 32, 64, 4, 4, stride=2, bias=True, leak=0.2, launches=2, tile=tile(32)),
      # launches the prefetch does not serve: an odd column count, a residual and a mask together
      fwd("fwd per-tap", 2, 17, 17, 32, 33, 3, 3, bias=True, residual=True, opts=NO_HALO, launches=2, tile=tile(ep=0)),
      fwd("fwd per-tap", 2, 9, 16, 32, 64, 3, 3, bias=True, residual=True, leak=0.2, opts=NO_HALO, launches=2,
          tile=tile(ep=0)),
  ]


def sm_count():
  return torch.cuda.get_device_properties(0).multi_processor_count


def ids(cs):
  return [c.id.replace("-n%d-" % c.n, "-nSM-") for c in cs]


def plain(c):
  """The case without any epilogue operand."""
  return Case(c.path, c.op, c.n, c.h, c.w, c.cin, c.cout, c.kh, c.kw, c.stride, c.up, c.pad, opts=c.opts,
              launches=c.launches, tile={k: v for k, v in c.tile.items() if k != EP})


def algebra(c, y0, ex, round_out):
  """The register epilogue's fp32 arithmetic applied to y0, in its order."""
  f = np.float32
  y = y0
  if "bias" in ex:
    y = (y + ex["bias"]).astype(f)
  if "residual" in ex:
    y = (y + ex["residual"]).astype(f)
  if c.relu:
    y = np.maximum(y, f(0))
  if "mask" in ex:
    y = relu_gate(ex["mask"], y, c.leak)
  return rna_tf32(y) if round_out else y


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(cases(132))), ids=ids(cases(132)))
def test_prefetched_epilogue_operands(K, i):
  """Element-wise against float64 (two runs bit-identical, the reported geometry and epilogue asserted), then bit for
  bit the fp32 algebra over the launch without epilogue operands, stored as is and TF32-rounded."""
  c = cases(sm_count())[i]
  check_case(K, c)
  a, b, ex = draw(c)
  p = plain(c)
  y0, launched, path = run(K, p, a, b, {})
  assert_path(K, p, launched, path)
  assert K.lib().get_option(EP) == 0
  for round_out in (False, True):
    y, launched, path = run(K, c, a, b, ex, round_out=round_out)
    assert_path(K, c, launched, path)
    assert same_bits(y, algebra(c, y0, ex, round_out)), "%s: epilogue differs from its fp32 algebra (round_out %s)" % (
        c.id, round_out)


@pytest.mark.gpu
@pytest.mark.parametrize("kh,kw,stride,pad", [(3, 3, 1, "SAME"), (3, 3, 2, "VALID")])
def test_prefetched_residual_into_a_channel_slice(K, kh, kw, stride, pad):
  """A forward convolution stored into channels [24, 24 + cout) of a wider NHWC tensor, its residual read from the same
  slice of a tensor of that width: element-wise exact, bit-identical to the dense launch, the neighbouring channels keep
  their bits, and the residual was prefetched."""
  c = fwd("fwd sliced", 2, 13, 10, 32, 36, kh, kw, stride=stride, pad=pad, bias=True, residual=True, relu=True,
          opts=NO_HALO, launches=2, tile=tile(64))
  ld, off = c.cout + 40, 24
  a, b, ex = draw(c)
  y64, scale = reference(c, a, b, ex)
  oh, ow = out_hw(c)
  rng = np.random.RandomState(1)
  fill = rng.standard_normal((c.n, oh, ow, ld)).astype(np.float32)
  wide_res = rng.standard_normal((c.n, oh, ow, ld)).astype(np.float32)
  wide_res[..., off:off + c.cout] = ex["residual"]
  dense = run(K, c, a, b, ex)[0]
  assert K.lib().get_option(EP) == 1
  lib = K.lib()
  A, B, bias, res = K.from_numpy(a), K.from_numpy(b), K.from_numpy(ex["bias"]), K.from_numpy(wide_res)
  buf = K.from_numpy(fill)
  n0 = lib.launch_count()
  with options(K, c.opts):
    ep = _lib.ConvEpilogue(bias.ptr, res.ptr + 4 * off, None, 0.0, _lib.CONV_RELU, ld)
    K._call("conv2d_fwd_ex", ctypes.byref(desc(K, c)), A.ptr, B.ptr, ctypes.byref(ep), buf.ptr + 4 * off)
  assert_path(K, c, lib.launch_count() - n0, _lib.PATH_NAMES[lib.get_option(_lib.OPT_LAST_PATH)])
  got = np.array(buf.cpu(), copy=True)
  check(got[..., off:off + c.cout], y64, scale, c.id + "-slice")
  assert same_bits(got[..., off:off + c.cout], dense), "sliced and dense outputs differ"
  assert np.array_equal(got[..., :off].view(np.uint32), fill[..., :off].view(np.uint32))
  assert np.array_equal(got[..., off + c.cout:].view(np.uint32), fill[..., off + c.cout:].view(np.uint32))


def test_cases_cover_the_prefetch_edges():
  """Without a GPU: the cases reach the edges the docstring names, at the H100's 132 SMs and at a smaller part's."""
  for sms in (132, 114):
    cs = cases(sms)
    assert len(set(ids(cs))) == len(cs)
    assert any(c.h == 17 and c.tile[EP] for c in cs) and any(c.h == 35 and c.tile[EP] for c in cs)
    assert any(c.tile.get(_lib.OPT_LAST_TC_MT) == 2 and c.tile.get(_lib.OPT_LAST_TC_BN) == 64 for c in cs)
    assert any(c.tile.get(_lib.OPT_LAST_TC_BN) == 256 and c.tile.get(_lib.OPT_LAST_TC_CTAS_PER_SM) == 1 for c in cs)
    assert any(c.op == "dgrad" and c.up and c.leak is not None and c.tile[EP] for c in cs)
    assert any(c.op == "dgrad" and c.stride == 2 and c.leak is not None and c.tile[EP] for c in cs)
    assert any(not c.tile[EP] for c in cs)
