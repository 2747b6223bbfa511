"""TEST INFRASTRUCTURE ONLY: the reference's fractal dimension (reference metrics/fractal_dimension.py:39-97) restated
in numpy / scipy: cdist of every sample to the seeds, bin edges spaced geometrically between the smallest non-zero and
the largest distance, N(r) from np.less.outer, and the least-squares slope of log N(r) against log r around the middle
of the log N range.  The seed indices can be injected; it also backs the emulated C-ABI entries of
tests/test_fractal_dimension.py."""
import numpy as np
import scipy.spatial


def distances(points, seeds):
  """[n, s] float64 Euclidean distances (scipy's cdist, summed sequentially over D)."""
  return scipy.spatial.distance.cdist(np.asarray(points, np.float64), np.asarray(seeds, np.float64))


def edges(flat, n_bins):
  """The n_bins geometric bin edges of the distances `flat`."""
  lo = np.min(flat[np.nonzero(flat)])
  hi = np.max(flat)
  return lo * ((hi / lo) ** np.linspace(0, 1, n_bins))


def counts(flat, upper, chunk=1 << 17):
  """N(r) for every edge r in `upper`: the distances strictly below it.  np.less.outer over chunks of the distances
  (integer sums, so equal to one outer product over all of them, without its N*S x n_bins bytes)."""
  return sum(np.sum(np.less.outer(flat[q:q + chunk], upper), axis=0) for q in range(0, len(flat), chunk))


def slope_from_distances(dist, n_bins=1000, scale=0.1):
  """The fit of the reference on an [n, s] distance table."""
  n, s = dist.shape
  flat = np.asarray(dist, np.float64).ravel()
  buckets = edges(flat, n_bins)
  table = np.zeros((n_bins - 1, 2))
  table[:, 0] = buckets[1:]
  table[:, 1] = counts(flat, buckets[1:])
  top, bottom = np.log(n * s), np.log(s)
  with np.errstate(divide="ignore"):
    x, y = np.log(table[:, 0]), np.log(table[:, 1])
  width = top - bottom
  mid = bottom + 0.5 * width
  lo = np.argmax(y > mid - scale * width)
  hi = np.argmax(y > mid + scale * width)
  design = np.vstack([x[lo:hi], np.ones(hi - lo)]).transpose()
  return np.linalg.lstsq(a=design, b=y[lo:hi].reshape(hi - lo, 1))[0][0][0]


def fractal_dimension(images, seed_idx, n_bins=1000, scale=0.1):
  """The reference's compute_fractal_dimension with the seed rows given: images [N, ...], seed_idx [S]."""
  flat = np.reshape(np.asarray(images), (len(images), -1))
  return slope_from_distances(distances(flat, flat[np.asarray(seed_idx)]), n_bins, scale)
