"""The tensor-core filter gradient (csrc/wgrad_tc.cu) with its activation operand fed to wgmma from registers: every
thread loads its A fragments (ci rows x pixels) straight out of the 128B-swizzled TMA stage, and only dY is transposed
through shared memory.  The cases cover what that changes: the row-to-channel mapping of the fragments and the
epilogue at every column-tile width, a ci tile hanging over Cin, the CTA past the last (tap, ci-tile) unit at two units
per CTA (no MMAs for the absent unit), the zeroed pixel rows of boxes of fewer than 32 pixels, the up-sampling views
of dY, operands rounded in the kernel or flagged as already rounded, and the per-image launch of the batched GEMM.

Each case is checked element by element against float64 on TF32-exact operands with the criterion of
test_tc_exact_gpu.py (|y - y64| <= TAU * A, A the contraction over |operands|), and run twice for bit-identical
results."""
import numpy as np
import pytest

from compare_gan_b200 import _lib
from tests.test_tc_exact_gpu import Case, assert_path, check, draw, options, reference, run, same_bits, wgrad

pytestmark = pytest.mark.gpu

MT1 = {_lib.OPT_TC_MT: 1}
MT2 = {_lib.OPT_TC_MT: 2}

CASES = [
    # 3x3 over one ci tile: 9 units, so at two units per CTA the fifth tile holds one
    wgrad("wgrad", 4, 16, 16, 128, 128, 3, 3, opts=MT2, note="9units-mt2"),
    wgrad("wgrad", 4, 16, 16, 128, 128, 3, 3, opts=MT1, note="9units-mt1"),
    # column-tile widths 32 / 96 / 128 at two units per CTA, 160 / 256 (one unit per CTA) and 96 at one
    wgrad("wgrad", 4, 16, 16, 128, 32, 3, 3, opts=MT2, note="bn32"),
    wgrad("wgrad", 4, 16, 16, 128, 96, 3, 3, opts=MT2, note="bn96"),
    wgrad("wgrad", 4, 16, 16, 128, 96, 3, 3, opts=MT1, note="bn96-mt1"),
    wgrad("wgrad", 4, 8, 8, 256, 128, 3, 3, opts=MT2, note="bn128"),
    wgrad("wgrad", 4, 8, 8, 128, 160, 3, 3, note="bn160"),
    wgrad("wgrad", 4, 8, 8, 128, 256, 3, 3, note="bn256"),
    # a ci tile hanging over Cin (96 = 0.75 tile; 160 = 1.25 tiles), at one and two units per CTA
    wgrad("wgrad", 4, 16, 16, 96, 64, 3, 3, opts=MT2, note="cin96"),
    wgrad("wgrad", 4, 16, 16, 160, 64, 3, 3, opts=MT2, note="cin160"),
    wgrad("wgrad", 4, 16, 16, 160, 128, 3, 3, opts=MT1, note="cin160-mt1"),
    # grids whose width neither divides 32 nor is a multiple of it: boxes of fewer than 32 pixels (zeroed tail rows)
    wgrad("wgrad", 2, 48, 48, 64, 64, 3, 3, note="w48"),
    wgrad("wgrad", 4, 24, 24, 64, 128, 3, 3, note="w24"),
    wgrad("wgrad", 4, 12, 12, 128, 64, 3, 3, note="w12"),
    wgrad("wgrad", 8, 6, 6, 64, 64, 3, 3, note="w6"),
    wgrad("wgrad", 4, 3, 3, 128, 128, 3, 3, note="w3"),
    # a conv over the zero-inserted 2x up-sampled input: four phase views of dY
    wgrad("wgrad", 4, 8, 8, 128, 128, 3, 3, up=True, note="up"),
    wgrad("wgrad", 4, 8, 8, 128, 128, 1, 1, up=True, note="up-1x1"),
]


@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  kernels.set_math_mode(1)
  yield kernels
  kernels.set_math_mode(0)


@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_wgrad_register_operand_elementwise(K, c):
  a, b, ex = draw(c)
  y64, scale = reference(c, a, b, ex)
  rounded, launched, path = run(K, c, a, b, ex)
  assert_path(K, c, launched, path)
  check(rounded, y64, scale, c.id)
  again = run(K, c, a, b, ex)[0]
  assert same_bits(rounded, again), "%s: two runs differ" % c.id
  # both operands flagged as TF32 values: the kernel skips the A-fragment and dY rounding, with the same bits
  flagged = run(K, c, a, b, ex, wflags=_lib.CONV_IN_TF32 | _lib.CONV_IN2_TF32)[0]
  assert same_bits(rounded, flagged), "%s: pre-rounded operands give other bits" % c.id


PER_IMAGE = [
    Case("bmm tn", "bmm_tn", 4, 64, 128, 256, 0, launches=1, note="per-image"),
    Case("bmm tn", "bmm_tn", 3, 96, 256, 512, 0, launches=1, note="per-image"),
]


@pytest.mark.parametrize("c", PER_IMAGE, ids=[c.id for c in PER_IMAGE])
def test_wgrad_register_operand_per_image(K, c):
  """C[i] = A[i]^T B[i] of the batched GEMM: the filter-gradient kernel with one image per split and no reduction."""
  a, b, ex = draw(c)
  y64, scale = reference(c, a, b, ex)
  got, launched, path = run(K, c, a, b, ex)
  assert_path(K, c, launched, path)
  check(got, y64, scale, c.id)
  with options(K, MT1):
    assert same_bits(got, run(K, c, a, b, ex)[0]), "%s: two runs differ" % c.id
