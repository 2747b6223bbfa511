"""The staged epilogue of the per-tap wgmma convolution (tile_epilogue_smem in csrc/conv_tc.cu): every float2 launch with
at most one of residual / mask whose output TMA can address (16-byte aligned base, phase offsets and pixel strides)
finishes its tile in the stage ring and stores it by TMA through one output map per phase, which clips rows past the
grid or the phase's extent and columns past cout.

Each case is checked element by element against float64 by the criterion of test_tc_exact_gpu.py (two runs
bit-identical, the reported geometry asserted, CGAN_OPT_LAST_TC_TMA_STORE among it), and bit for bit against the fp32
algebra of its epilogue over the launch without any epilogue operand, stored as is and TF32-rounded.  The cases are the
bias-only and bare launches that the residual / mask prefetch of test_tc_epilogue_operands_gpu.py did not stage: 17x17
and 35x35 maps (boxes hanging over the grid), two pixel tiles per CTA at a 64-wide column tile with an odd tile count,
the 256-wide tile at one CTA per SM, 96- and 160-wide tiles, even column counts that are not a multiple of 32, the four
output phases of an up-sampling forward and a stride-2 input gradient over an odd grid (phases of unequal extent).  Two
cases carry a residual or a mask through the same ring.  An even column count that is not a multiple of 4 has 8-byte
pixel strides, which TMA cannot address: that launch reports the register epilogue.  Separate tests store into a
channel slice of a wider tensor (the dispatcher hands the kernel only slices at a multiple of 4 channels with a width
that is a multiple of 4, which TMA can address) and into the residual itself, in place."""
import ctypes

import numpy as np
import pytest
import torch

from compare_gan_b200 import _lib
from tests.test_tc_exact_gpu import (K, NO_HALO, assert_path, check, check_case, desc, dgrad, draw, fwd,  # noqa: F401
                                     mt2_batch, options, out_hw, out_shape, reference, run, same_bits)
from tests.test_tc_epilogue_operands_gpu import algebra, plain

TMA = _lib.OPT_LAST_TC_TMA_STORE
EP = _lib.OPT_LAST_TC_EP_SMEM


def tile(width=None, mt=None, ctas=None, tma=1, ep=0):
  t = {TMA: tma, EP: ep, _lib.OPT_LAST_TC_HALO: 0}
  for key, v in ((_lib.OPT_LAST_TC_BN, width), (_lib.OPT_LAST_TC_MT, mt), (_lib.OPT_LAST_TC_CTAS_PER_SM, ctas)):
    if v is not None:
      t[key] = v
  return t


def cases(sms):
  two, mt2 = 2 * sms, mt2_batch(sms)
  return [
      # boxes hanging over the grid: 17x7 and 35x3 boxes, bias only and bare, with and without ReLU
      fwd("fwd per-tap", 2, 17, 17, 32, 64, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=tile(64)),
      fwd("fwd per-tap", 2, 17, 17, 32, 64, 3, 3, bias=True, relu=True, opts=NO_HALO, launches=2, tile=tile(64)),
      fwd("fwd per-tap", 2, 35, 35, 32, 64, 3, 3, opts=NO_HALO, launches=2, tile=tile(64)),
      fwd("fwd per-tap", 2, 35, 35, 32, 64, 3, 3, relu=True, opts=NO_HALO, launches=2, tile=tile(64)),
      dgrad("dgrad per-tap", 2, 17, 17, 64, 64, 3, 3, launches=2, tile=tile(64)),
      dgrad("dgrad per-tap", 2, 35, 35, 64, 32, 3, 3, bias=True, launches=2, tile=tile(64)),
      # two pixel tiles per CTA at bn = 64, an odd tile count: the last CTA stores its first tile only
      fwd("fwd per-tap", mt2, 8, 8, 32, 64, 3, 3, bias=True, relu=True, opts=NO_HALO, launches=2, note="mt2-odd",
          tile=tile(64, mt=2, ctas=2)),
      dgrad("dgrad per-tap", mt2, 8, 8, 64, 64, 3, 3, opts=NO_HALO, launches=2, note="mt2-odd",
            tile=tile(64, mt=2, ctas=2)),
      # 256 columns: the 128-wide tile at two CTAs per SM, the 256-wide tile at one (eight chunks per CTA)
      fwd("fwd per-tap", two, 8, 16, 256, 256, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=tile(128, mt=1, ctas=2)),
      dgrad("dgrad per-tap", two, 8, 16, 256, 256, 3, 3, opts=NO_HALO, launches=2, tile=tile(128, mt=1, ctas=2)),
      fwd("fwd per-tap", two, 8, 16, 352, 256, 3, 3, bias=True, relu=True, opts=NO_HALO, launches=2, note="long-k",
          tile=tile(256, mt=1, ctas=1)),
      dgrad("dgrad per-tap", two - 1, 8, 16, 256, 128, 3, 3, opts=NO_HALO, launches=2, note="below-2-waves",
            tile=tile(256, mt=1, ctas=1)),
      # three- and five-chunk tiles
      fwd("fwd per-tap", 2, 9, 16, 64, 96, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=tile(96)),
      fwd("fwd per-tap", 2, 9, 16, 64, 160, 3, 3, relu=True, opts=NO_HALO, launches=2, tile=tile(160)),
      # even column counts that are not a multiple of 32: the store clips the last chunk's columns
      fwd("fwd per-tap", 2, 13, 10, 32, 36, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=tile(64)),
      fwd("fwd per-tap", 2, 13, 10, 32, 20, 3, 3, bias=True, relu=True, opts=NO_HALO, launches=2, tile=tile(32)),
      dgrad("dgrad per-tap", 2, 11, 12, 48, 64, 3, 3, launches=2, tile=tile(64)),
      # phases: the four output phases of an up-sampling forward, a stride-2 input gradient of an odd grid (phases of
      # unequal extent) and of an even one
      fwd("fwd phases", 2, 6, 9, 32, 64, 4, 4, up=True, bias=True, launches=2, tile=tile(64)),
      fwd("fwd phases", 2, 5, 7, 32, 96, 3, 3, up=True, relu=True, launches=2, tile=tile(96)),
      dgrad("dgrad s2 phases", 2, 15, 11, 64, 32, 3, 3, stride=2, tile=tile(64)),
      dgrad("dgrad s2 phases", 2, 12, 16, 32, 64, 4, 4, stride=2, bias=True, launches=2, tile=tile(32)),
      # with a prefetched residual / mask (the same ring, loaded instead of handed over)
      fwd("fwd per-tap", 2, 17, 17, 32, 64, 3, 3, bias=True, residual=True, relu=True, opts=NO_HALO, launches=2,
          tile=tile(64, ep=1)),
      dgrad("dgrad s2 phases", 2, 15, 11, 64, 32, 3, 3, stride=2, leak=0.2, tile=tile(64, ep=1)),
      # 8-byte pixel strides: the register epilogue
      fwd("fwd per-tap", 2, 13, 10, 32, 18, 3, 3, bias=True, relu=True, opts=NO_HALO, launches=2, tile=tile(tma=0)),
      dgrad("dgrad per-tap", 2, 11, 12, 34, 64, 3, 3, launches=2, tile=tile(tma=0)),
  ]


def sm_count():
  return torch.cuda.get_device_properties(0).multi_processor_count


def ids(cs):
  return [c.id.replace("-n%d-" % c.n, "-nSM-") for c in cs]


def call(K, c, A, B, dev, out_ptr, round_out=False, ldy=0):
  """One launch of the case into `out_ptr`; returns the path it took."""
  lib = K.lib()
  n0 = lib.launch_count()
  with options(K, c.opts):
    ep = K._epilogue(dev.get("bias"), dev.get("residual"), dev.get("mask"), c.leak or 0.0, c.relu, round_out, ldy=ldy)
    K._call("conv2d_fwd_ex" if c.op == "fwd" else "conv2d_dgrad_ex", ctypes.byref(desc(K, c)), A.ptr, B.ptr,
            ctypes.byref(ep), out_ptr)
  return lib.launch_count() - n0, _lib.PATH_NAMES[lib.get_option(_lib.OPT_LAST_PATH)]


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(cases(132))), ids=ids(cases(132)))
def test_tma_stored_epilogue(K, i):
  """Element-wise against float64, then bit for bit the fp32 algebra over the launch without epilogue operands, stored
  as is and TF32-rounded."""
  c = cases(sm_count())[i]
  check_case(K, c)
  a, b, ex = draw(c)
  p = plain(c)
  p.tile = {**c.tile, EP: 0}
  y0, launched, path = run(K, p, a, b, {})
  assert_path(K, p, launched, path)
  for round_out in (False, True):
    y, launched, path = run(K, c, a, b, ex, round_out=round_out)
    assert_path(K, c, launched, path)
    assert same_bits(y, algebra(c, y0, ex, round_out)), "%s: epilogue differs from its fp32 algebra (round_out %s)" % (
        c.id, round_out)


@pytest.mark.gpu
@pytest.mark.parametrize("kh,kw,stride,pad,off,ld", [(3, 3, 1, "SAME", 24, 76), (3, 3, 2, "VALID", 4, 40)])
def test_channel_slice(K, kh, kw, stride, pad, off, ld):
  """A forward convolution (bias, ReLU) stored into channels [off, off + cout) of a tensor `ld` channels wide: element-
  wise exact, bit-identical to the dense launch, the neighbouring channels keep their bits (the store clips the box at
  cout), and the launch stored by TMA."""
  c = fwd("fwd sliced", 2, 13, 10, 32, 36, kh, kw, stride=stride, pad=pad, bias=True, relu=True, opts=NO_HALO,
          launches=2, tile=tile(64))
  a, b, ex = draw(c)
  y64, scale = reference(c, a, b, ex)
  oh, ow = out_hw(c)
  fill = np.random.RandomState(1).standard_normal((c.n, oh, ow, ld)).astype(np.float32)
  dense = run(K, c, a, b, ex)[0]
  assert K.lib().get_option(TMA) == 1
  buf = K.from_numpy(fill)
  launched, path = call(K, c, K.from_numpy(a), K.from_numpy(b), {"bias": K.from_numpy(ex["bias"])}, buf.ptr + 4 * off,
                        ldy=ld)
  assert_path(K, c, launched, path)
  got = np.array(buf.cpu(), copy=True)
  check(got[..., off:off + c.cout], y64, scale, c.id + "-slice")
  assert same_bits(got[..., off:off + c.cout], dense), "sliced and dense outputs differ"
  assert np.array_equal(got[..., :off].view(np.uint32), fill[..., :off].view(np.uint32))
  assert np.array_equal(got[..., off + c.cout:].view(np.uint32), fill[..., off + c.cout:].view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 17, 17, 32, 64), (2, 8, 16, 256, 256)])
def test_output_aliasing_its_residual(K, n, h, w, cin, cout):
  """out == residual, updated in place (every chunk of the residual is loaded before the store of the same chunk, and
  no other CTA touches it): bit-identical to the launch into a separate output."""
  c = fwd("fwd in place", n, h, w, cin, cout, 3, 3, bias=True, residual=True, relu=True, opts=NO_HALO, launches=2,
          tile=tile(ep=1))
  a, b, ex = draw(c)
  separate = run(K, c, a, b, ex)[0]
  res = K.from_numpy(ex["residual"])
  launched, path = call(K, c, K.from_numpy(a), K.from_numpy(b), {"bias": K.from_numpy(ex["bias"]), "residual": res},
                        res.ptr)
  assert_path(K, c, launched, path)
  assert same_bits(np.array(res.cpu(), copy=True), separate), "in-place and separate outputs differ"


def test_cases_cover_the_store_edges():
  """Without a GPU: the cases reach the edges the docstring names, at the H100's 132 SMs and at a smaller part's."""
  for sms in (132, 114):
    cs = cases(sms)
    assert len(set(ids(cs))) == len(cs)
    assert any(not c.tile[TMA] for c in cs)
    bare = [c for c in cs if not (c.bias or c.residual or c.leak is not None)]
    bias_only = [c for c in cs if c.bias and not (c.residual or c.leak is not None)]
    for group in (bare, bias_only):
      assert any(c.relu for c in group) and any(not c.relu for c in group)
    assert any(c.h == 17 for c in bare) and any(c.h == 35 for c in bare)
    assert any(c.tile.get(_lib.OPT_LAST_TC_MT) == 2 and c.tile.get(_lib.OPT_LAST_TC_BN) == 64 for c in cs)
    assert any(c.tile.get(_lib.OPT_LAST_TC_BN) == 256 and c.tile.get(_lib.OPT_LAST_TC_CTAS_PER_SM) == 1 for c in cs)
    assert {96, 160} <= {c.tile.get(_lib.OPT_LAST_TC_BN) for c in cs}
    assert any(out_shape(c)[-1] % 2 == 0 and out_shape(c)[-1] % 32 for c in cs)
    assert any(c.op == "fwd" and c.up for c in cs)
    assert any(c.op == "dgrad" and c.stride == 2 and c.h % 2 and c.w % 2 for c in cs)
