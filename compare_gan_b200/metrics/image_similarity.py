"""MS-SSIM of image pairs (reference metrics/image_similarity.py).  The O(pixels) work — pyramid, Gaussian filtering,
luminance and contrast-structure maps and their pixel means — runs on the device (cgan_ssim_terms); the O(pairs) tail —
relu, power factors, product over scales, mean over channels (image_similarity.py:323-332) — runs here in float64."""
import numpy as np

# a tuple so that it cannot be changed by accident (image_similarity.py:214-216)
_MSSSIM_WEIGHTS = (.0448, 0.2856, 0.3001, 0.2363, 0.1333)


def combine(terms, power_factors):
  """[pairs, levels, c] per-scale terms -> [pairs] MS-SSIM: prod over levels of relu(term)^power, mean over channels."""
  t = np.maximum(np.asarray(terms, np.float64), 0.0)
  return np.prod(t ** np.asarray(power_factors, np.float64)[None, :, None], axis=1).mean(axis=1)


def _device(images):
  from .. import kernels as K
  from ..tape import DT
  if isinstance(images, DT):
    return images
  return K.from_numpy(np.asarray(images, np.float32))


def pair_scores(images, pairs, power_factors=_MSSSIM_WEIGHTS, filter_size=11, filter_width=1.5, max_val=255.0):
  """MS-SSIM [npairs] float64 of the pairs (i, j) of one image set [n,h,w,c] (numpy or DT, values in [0, max_val])."""
  from .. import kernels as K
  terms = K.ssim_terms(_device(images), pairs, len(power_factors), filter_size, filter_width, max_val)
  return combine(terms, power_factors)


def _multiscale_ssim_helper(img1, img2, filter_size, filter_width, power_factors, max_val=255.0):
  """Per-element MS-SSIM of two equally shaped batches [B,h,w,c]: the pairs (k, B + k) of their concatenation."""
  a, b = np.asarray(img1, np.float32), np.asarray(img2, np.float32)
  if a.ndim != 4 or a.shape != b.shape:
    raise ValueError("two images are not compatible: %s and %s" % (a.shape, b.shape))
  bsz = a.shape[0]
  pairs = np.stack([np.arange(bsz), bsz + np.arange(bsz)], axis=1)
  return pair_scores(np.concatenate([a, b]), pairs, power_factors, filter_size, filter_width, max_val)


def multiscale_ssim(img1, img2, filter_size=11, filter_width=1.5, max_val=255.0):
  """MS-SSIM with the power factors of Wang et al. (image_similarity.py:219-226)."""
  return _multiscale_ssim_helper(img1, img2, filter_size, filter_width, _MSSSIM_WEIGHTS, max_val)


def multiscale_ssim_unweighted(img1, img2, filter_size=11, filter_width=1.5, max_val=255.0):
  """MS-SSIM with unit power factors (image_similarity.py:229-236)."""
  return _multiscale_ssim_helper(img1, img2, filter_size, filter_width, [1, 1, 1, 1, 1], max_val)
