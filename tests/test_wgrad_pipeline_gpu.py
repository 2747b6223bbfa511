"""The tensor-core filter gradient (csrc/wgrad_tc.cu) on shapes whose CTAs run long pixel loops.  Its consumer warpgroups
transpose k-block kb + 1 into one shared-memory buffer while the MMAs of kb read the other, so a missing or misplaced
barrier only shows after many k-blocks.  Each case runs the filter gradient twice and checks that the two results are
bit-identical and that both match a float64 evaluation on the same TF32-rounded operands."""
import numpy as np
import pytest
import torch

from tests.abi_emulator import rna_tf32
from tests.gpu_util import assert_close

pytestmark = pytest.mark.gpu

CASES = [
    # name, n, h, cin, cout, k, upsample
    ("biggan D 3x3 1536->1536 @4", 128, 4, 1536, 1536, 3, False),      # one split: 64 k-blocks per CTA
    ("cifar G 3x3 256->256 @32", 64, 32, 256, 256, 3, False),          # 147 k-blocks per CTA, 256-wide column tile
    ("cifar G 3x3 256->256 up 16->32", 64, 16, 256, 256, 3, True),     # sub-pixel phase views of dY
    ("cifar D 3x3 128->128 @32", 128, 32, 128, 128, 3, False),         # two (tap, ci-tile) units per CTA
]


@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  return kernels


def wgrad_f64(x, dy, k, up):
  """dW[kh, kw, ci, co] in float64 for a stride-1 SAME conv (over the zero-inserted 2x input when `up`)."""
  xt = torch.from_numpy(x).cuda().double()
  if up:
    n, h, w, c = xt.shape
    z = torch.zeros(n, 2 * h, 2 * w, c, dtype=torch.float64, device=xt.device)
    z[:, ::2, ::2, :] = xt
    xt = z
  g = torch.from_numpy(dy).cuda().double()
  gw = torch.nn.grad.conv2d_weight(xt.permute(0, 3, 1, 2), (dy.shape[3], x.shape[3], k, k), g.permute(0, 3, 1, 2),
                                   padding=(k - 1) // 2)
  return gw.permute(2, 3, 1, 0).cpu().numpy()


@pytest.mark.parametrize("name,n,h,cin,cout,k,up", CASES, ids=[c[0] for c in CASES])
def test_wgrad_long_loops_repeatable_and_exact(K, name, n, h, cin, cout, k, up):
  rng = np.random.RandomState(sum(map(ord, name)))
  oh = 2 * h if up else h
  x = rng.standard_normal((n, h, h, cin)).astype(np.float32)
  dy = rng.standard_normal((n, oh, oh, cout)).astype(np.float32)
  d = K.conv_desc(n, h, h, cin, cout, k, k, 1, up, "SAME")
  K.set_math_mode(1)
  try:
    xd, dyd = K.from_numpy(x), K.from_numpy(dy)
    first = np.array(K.conv2d_wgrad(d, xd, dyd).cpu(), copy=True)
    second = np.array(K.conv2d_wgrad(d, xd, dyd).cpu(), copy=True)
  finally:
    K.set_math_mode(0)
  assert first.shape == (k, k, cin, cout)
  assert np.array_equal(first.view(np.uint32), second.view(np.uint32)), "%s: two runs differ" % name
  ref = wgrad_f64(rna_tf32(x), rna_tf32(dy), k, up)
  assert_close(first, ref, 1e-4, "%s wgrad vs float64 on TF32 operands" % name)
