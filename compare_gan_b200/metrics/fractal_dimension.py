"""Fractal dimension of a generated set (reference metrics/fractal_dimension.py): the slope of log N(r) against log r,
N(r) being the number of (sample, seed) pairs closer than r, fitted around the middle of the log N range.

The N x S seed distances are computed on the device in float64 (csrc/fractal.cu), and so are their range and the
counts below each bin edge; the bin edges, logs, argmax and least-squares fit are the reference's numpy expressions in
float64 on the host.  Deliberate differences from the reference:
  - inside `evaluate` the seeds are the first S generated samples of each averaging run (distinct i.i.d. draws from G),
    not a draw with replacement from NumPy's global RNG after the whole set exists: the distances are streamed batch by
    batch, so the seeds must exist before the rest of the set.  The score of a given set and seed choice is pinned,
    which samples become seeds is not.  `compute_fractal_dimension` draws its seeds as the reference does;
  - every averaging run is scored; the reference keeps the images of the first run only (eval_gan_lib.py:179-183), so
    with num_averaging_runs > 1 its task cannot run;
  - the squared differences are summed in a fixed slice order over D, not sequentially as scipy's cdist does; the
    distances differ by far less than the float64 resolution of a bin edge, but not by zero;
  - the points are fp32 (the reference's images are float32), and a set whose distances are all 0 raises a ValueError
    that names the cause."""
import numpy as np

from . import eval_task


def _random_state(random_state):
  if random_state is None:
    return np.random.mtrand._rand
  if isinstance(random_state, np.random.RandomState):
    return random_state
  return np.random.RandomState(random_state)


def _check_shape(shape, num_fd_seeds):
  if len(shape) < 2 or shape[0] < num_fd_seeds:
    raise ValueError("the fractal dimension needs an [N, ...] array of N >= num_fd_seeds = %d samples, got shape %s"
                     % (num_fd_seeds, tuple(shape)))


def fractal_dimension_from_distances(dist, n, s, n_bins=1000, scale=0.1):
  """The reference's tail (fractal_dimension.py:69-97) on the distances of n samples to s seeds, a contiguous
  [n, s] float64 device tensor."""
  from .. import kernels as K
  min_distance, max_distance = K.fd_range(dist)
  if not np.isfinite(max_distance):
    raise ValueError("the seed distances are not finite: the samples hold NaN or inf")
  if min_distance == np.inf:
    raise ValueError("every seed distance is 0: all samples are identical, so the fractal dimension is undefined")
  buckets = min_distance * ((max_distance / min_distance) ** np.linspace(0, 1, n_bins))
  fd_result = np.zeros((n_bins - 1, 2))
  fd_result[:, 0] = buckets[1:]
  fd_result[:, 1] = K.fd_counts(dist, buckets[1:])
  max_y = np.log(n * s)
  min_y = np.log(s)
  with np.errstate(divide="ignore"):      # log N(r) of the empty bins below the nearest pair is -inf, as in the reference
    x = np.log(fd_result[:, 0])
    y = np.log(fd_result[:, 1])
  y_width = max_y - min_y
  y_val = min_y + 0.5 * y_width
  start = np.argmax(y > y_val - scale * y_width)
  end = np.argmax(y > y_val + scale * y_width)
  a = np.vstack([x[start:end], np.ones(end - start)]).transpose()
  return np.linalg.lstsq(a=a, b=y[start:end].reshape(end - start, 1))[0][0][0]


def compute_fractal_dimension(fake_images, num_fd_seeds=100, n_bins=1000, scale=0.1, random_state=None):
  """Fractal dimension of fake_images [N, ...] (numpy or a device DT; any scaling), from num_fd_seeds seed samples
  drawn with replacement by `random_state` (None: NumPy's global state, as the reference's np.random.randint)
  (reference fractal_dimension.py:39-97)."""
  import torch
  from .. import kernels as K
  from ..tape import DT
  _check_shape(fake_images.shape, num_fd_seeds)
  n = int(fake_images.shape[0])
  if isinstance(fake_images, DT):
    x = fake_images.t.reshape(n, -1).float().contiguous()
  else:
    x = torch.from_numpy(np.ascontiguousarray(np.asarray(fake_images, np.float32).reshape(n, -1))).to(K._RT["device"])
  idx = _random_state(random_state).randint(n, size=num_fd_seeds)
  seeds = x[torch.from_numpy(idx).to(x.device)].contiguous()
  dist = K.fd_distances(x, seeds)
  return fractal_dimension_from_distances(dist, n, num_fd_seeds, n_bins, scale)


class FractalDimensionTask(eval_task.EvalTask):
  """Fractal dimension of each averaging run's generated set, seeded by its first num_fd_seeds samples (x255, as the
  reference's images).  In a sharded evaluation it comes from rank 0's shard and is broadcast, so every rank returns the
  same value."""
  _LABEL = "fractal_dimension"

  def __init__(self, num_fd_seeds=100, n_bins=1000, scale=0.1):
    self.num_fd_seeds, self.n_bins, self.scale = int(num_fd_seeds), int(n_bins), float(scale)
    self.distance_seeds = self.num_fd_seeds
    self.images_needed = self.num_fd_seeds

  def metric_list(self):
    return frozenset([self._LABEL])

  def _score(self, fake_dset):
    dist = getattr(fake_dset, "seed_distances", None)
    if dist is None or dist.shape[1] < self.num_fd_seeds:
      raise ValueError("the fractal dimension needs N >= num_fd_seeds = %d generated samples with their seed distances"
                       % self.num_fd_seeds)
    dist = dist[:, :self.num_fd_seeds].contiguous()
    return float(fractal_dimension_from_distances(dist, dist.shape[0], self.num_fd_seeds, self.n_bins, self.scale))

  def run_after_session(self, fake_dset, real_dset):
    del real_dset
    from ..tpu import tpu_ops
    if tpu_ops.num_replicas() == 1:
      return {self._LABEL: self._score(fake_dset)}
    import torch
    import torch.distributed as dist
    from .. import kernels as K
    score, error = float("nan"), ""
    if dist.get_rank() == 0:
      try:
        score = self._score(fake_dset)
      except ValueError as e:
        error = str(e)            # raised on every rank below, after the broadcast
    t = torch.tensor([score], dtype=torch.float64, device=K._RT["device"])
    dist.broadcast(t, 0)
    score = float(t.item())
    if np.isnan(score):
      raise ValueError(error or "the fractal dimension of rank 0's samples is undefined")
    return {self._LABEL: score}
