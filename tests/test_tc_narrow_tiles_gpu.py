"""The 128-wide column tile that the per-tap wgmma convolution takes for 256-column outputs on large grids with short K
loops (tc_pick_bn_per_tap in csrc/conv_tc.cu): every launch class of the generator's 256-channel layers that now runs
it, element by element against float64 by the criterion of test_tc_exact_gpu.py, with the geometry the launch reports
(column tile, pixel tiles per CTA, per-tap kernel, and two CTAs per SM from the CUDA occupancy calculator).  A long K
loop and a one-wave grid keep the 256-wide tile.

The batches are sized from the SM count: on 8x16 maps a pixel tile is one image, on 4x8 maps four, so 2 x SMs tiles
make the two waves of 256-wide CTAs the rule asks for."""
import pytest
import torch

from compare_gan_b200 import _lib
from tests.test_tc_exact_gpu import K, NO_HALO, check_case, dgrad, fwd  # noqa: F401  (K: the module's fixture)


def geometry(width, ctas_per_sm):
  return {_lib.OPT_LAST_TC_BN: width, _lib.OPT_LAST_TC_MT: 1, _lib.OPT_LAST_TC_HALO: 0,
          _lib.OPT_LAST_TC_CTAS_PER_SM: ctas_per_sm}


def narrow_cases(sms):
  two = 2 * sms
  narrow = geometry(128, 2)
  return [
      # G's 3x3 256->256 convolutions (72 k-blocks) and their input gradients
      fwd("fwd per-tap", two, 8, 16, 256, 256, 3, 3, bias=True, relu=True, opts=NO_HALO, launches=2, tile=narrow),
      dgrad("dgrad per-tap", two, 8, 16, 256, 256, 3, 3, bias=True, leak=0.0, opts=NO_HALO, launches=2, tile=narrow),
      # the 2x upsampling 3x3 convolution: four sub-pixel phases of 4, 2, 2 and 1 taps in one launch, and its input
      # gradient (9 taps over the four parity views of dy)
      fwd("fwd phases", 4 * sms, 4, 8, 256, 256, 3, 3, up=True, bias=True, residual=True, launches=2, tile=narrow),
      dgrad("dgrad phases", two, 8, 16, 256, 256, 3, 3, up=True, leak=0.2, launches=2, tile=narrow),
      # the 1x1 upsampling shortcut: phase 0 on the tensor cores, the bias-only phases, the post pass
      fwd("fwd 1x1-up", two, 8, 16, 256, 256, 1, 1, up=True, bias=True, launches=3, tile=narrow),
      # 512 columns: two 128-wide column tiles per 256 columns of the wide rule
      fwd("fwd per-tap", sms, 8, 16, 128, 512, 3, 3, bias=True, opts=NO_HALO, launches=2, tile=narrow),
  ]


def wide_cases(sms):
  two = 2 * sms
  return [
      # 11 channel chunks x 9 taps = 99 k-blocks: the long K loop keeps the 256-wide tile (one CTA per SM)
      fwd("fwd per-tap", two, 8, 16, 352, 256, 3, 3, bias=True, opts=NO_HALO, launches=2, note="long-k",
          tile=geometry(256, 1)),
      # fewer than two waves of 256-wide CTAs keep it too
      fwd("fwd per-tap", two - 1, 8, 16, 128, 256, 3, 3, bias=True, opts=NO_HALO, launches=2, note="below-2-waves",
          tile=geometry(256, 1)),
  ]


def sm_count():
  return torch.cuda.get_device_properties(0).multi_processor_count


def ids(cases):
  return [c.id.replace("-n%d-" % c.n, "-nSM-") for c in cases]


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(narrow_cases(132))), ids=ids(narrow_cases(132)))
def test_narrow_column_tile_elementwise(K, i):
  """Each launch class the 128-wide tile now serves: element-wise against float64, two runs bit-identical, and the
  launch reports bn 128, one pixel tile per CTA, the per-tap kernel and two CTAs per SM."""
  check_case(K, narrow_cases(sm_count())[i])


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(wide_cases(132))), ids=ids(wide_cases(132)))
def test_wide_column_tile_kept_elementwise(K, i):
  """Where the rule keeps the 256-wide tile (long K loop, or fewer than two waves): element-wise against float64, with
  the geometry asserted."""
  check_case(K, wide_cases(sm_count())[i])


def test_rule_cases_are_sized_for_the_rule():
  """Without a GPU: the cases above sit on the side of the rule they are meant for, at the H100's 132 SMs and at a
  smaller part's count (tile counts from tc_geometry: one image per tile on 8x16 maps, four on 4x8; k-blocks = taps of
  the longest phase x 32-channel chunks)."""
  for sms in (132, 114):
    for c in narrow_cases(sms) + wide_cases(sms):
      tiles = c.n if c.h == 8 else c.n // 4
      phases = 4 if (c.up and c.kh == 3 and c.op == "fwd") else 1
      taps = 4 if phases == 4 else c.kh * c.kw
      kchunks = -(-(c.cin if c.op == "fwd" else c.cout) // 32)
      cols = c.cout if c.op == "fwd" else c.cin
      waves = tiles * (cols // 256) * phases / float(sms)
      narrow = c.tile[_lib.OPT_LAST_TC_BN] == 128
      assert narrow == (waves >= 2 and taps * kchunks <= 96), (c.id, waves, taps * kchunks)
  assert len(set(ids(narrow_cases(132) + wide_cases(132)))) == len(narrow_cases(132) + wide_cases(132))
