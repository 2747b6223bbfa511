"""Float64 NumPy restatement of the reference's MS-SSIM (metrics/image_similarity.py, metrics/ms_ssim_score.py), written
literally: the softmax-normalised 2-D window of f_special_gauss, a VALID depthwise correlation with the full 2-D window,
the min(filter_size, h, w) clamp, SYMMETRIC padding of odd sides before the 2x2 average pool, compensation = 1, relu on
every cs and on the last ssim, and the ordered-pair sum minus B of compute_msssim."""
import numpy as np

K1, K2 = 0.01, 0.03
WEIGHTS = (.0448, 0.2856, 0.3001, 0.2363, 0.1333)


def f_special_gauss(size, sigma):
  """image_similarity.py:140-154: softmax over the flattened size x size grid of -(i^2 + j^2) / (2 sigma^2)."""
  coords = np.arange(size, dtype=np.float64) - (size - 1) / 2.0
  g = coords ** 2 * (-0.5 / sigma ** 2)
  g = (g[None, :] + g[:, None]).reshape(-1)
  e = np.exp(g - g.max())
  return (e / e.sum()).reshape(size, size)


def _reducer(x, kernel):
  """tf.nn.depthwise_conv2d(x, kernel tiled over channels, VALID) on [..., h, w, c]."""
  f = kernel.shape[0]
  win = np.lib.stride_tricks.sliding_window_view(x, (f, f), axis=(-3, -2))     # [..., oh, ow, c, f, f]
  return np.tensordot(win, kernel, axes=([-2, -1], [0, 1]))


def _ssim_per_channel(img1, img2, filter_size, filter_width, max_val):
  """image_similarity.py:85-211: (mean of luminance*cs, mean of cs) per channel, [..., c]."""
  size = min(filter_size, img1.shape[-3], img1.shape[-2])
  kernel = f_special_gauss(size, filter_width).astype(img1.dtype)
  c1, c2 = (K1 * max_val) ** 2, (K2 * max_val) ** 2
  mean0, mean1 = _reducer(img1, kernel), _reducer(img2, kernel)
  num0 = mean0 * mean1 * 2.0
  den0 = mean0 ** 2 + mean1 ** 2
  luminance = (num0 + c1) / (den0 + c1)
  num1 = _reducer(img1 * img2, kernel) * 2.0
  den1 = _reducer(img1 ** 2 + img2 ** 2, kernel)
  cs = (num1 - num0 + c2) / (den1 - den0 + c2)
  return (luminance * cs).mean(axis=(-3, -2)), cs.mean(axis=(-3, -2))


def _downscale(x):
  """SYMMETRIC pad of one row / column at the end of odd sides, then 2x2 VALID average pooling (:284-316)."""
  h, w = x.shape[-3], x.shape[-2]
  pad = [(0, 0)] * (x.ndim - 3) + [(0, h % 2), (0, w % 2), (0, 0)]
  x = np.pad(x, pad, mode="symmetric")
  h, w = x.shape[-3], x.shape[-2]
  return x.reshape(x.shape[:-3] + (h // 2, 2, w // 2, 2, x.shape[-1])).mean(axis=(-4, -2))


def terms(img1, img2, levels=5, filter_size=11, filter_width=1.5, max_val=255.0, dtype=np.float64):
  """[..., levels, c]: mean cs at levels 0..levels-2 and mean luminance*cs at the last level, before the relu — what
  cgan_ssim_terms returns per pair.  dtype=np.float32 gives a literal fp32 restatement (what fp32 rounding costs)."""
  a, b = np.asarray(img1, dtype), np.asarray(img2, dtype)
  out = []
  for k in range(levels):
    if k > 0:
      a, b = _downscale(a), _downscale(b)
    ssim, cs = _ssim_per_channel(a, b, filter_size, filter_width, max_val)
    out.append(ssim if k == levels - 1 else cs)
  return np.stack(out, axis=-2)


def multiscale_ssim(img1, img2, filter_size=11, filter_width=1.5, max_val=255.0, power_factors=WEIGHTS):
  """image_similarity.py:239-333: [...] MS-SSIM."""
  t = np.maximum(terms(img1, img2, len(power_factors), filter_size, filter_width, max_val), 0.0)
  return np.prod(t ** np.asarray(power_factors, np.float64)[:, None], axis=-2).mean(axis=-1)


def multiscale_ssim_unweighted(img1, img2, filter_size=11, filter_width=1.5, max_val=255.0):
  return multiscale_ssim(img1, img2, filter_size, filter_width, max_val, power_factors=[1, 1, 1, 1, 1])


def compute_msssim(images, num_batches):
  """ms_ssim_score.py:70-111 over consecutive batches: (sum over the B^2 ordered pairs - B) / (B^2 - B), averaged."""
  images = np.asarray(images, np.float64)
  bsz = images.shape[0] // num_batches
  assert bsz > 1
  scores = []
  for i in range(num_batches):
    batch = images[i * bsz:(i + 1) * bsz]
    pair1 = np.tile(batch, (bsz, 1, 1, 1))
    pair2 = np.repeat(batch, bsz, axis=0)
    score = multiscale_ssim(pair1, pair2).sum() - bsz
    scores.append(score / (bsz * bsz - bsz))
  return float(np.mean(scores))
