"""Precision and recall of a generative model (reference metrics/prd_score.py; Sajjadi et al., "Assessing Generative
Models via Precision and Recall", 2018).  The union of both embeddings is clustered, each set becomes a histogram over
the clusters, and the PRD curve of the two histograms says whether the model drops modes (low recall) or produces
samples off the data manifold (low precision).

The clustering runs on the device in float64 (csrc/kmeans.cu); the curves are the reference's formulas, in float64 on
the host.  Deliberate differences from the reference's sklearn MiniBatchKMeans(n_clusters, n_init=10):
  - full-batch Lloyd (the algorithm mini-batch k-means approximates) instead of mini-batch updates, so that a
    clustering is pinned by its random numbers: per averaging run, the best of n_init plain k-means++ seedings over all
    points (by inertia), then one Lloyd run from it, stopping as sklearn KMeans(algorithm="lloyd") does (unchanged
    labels, total squared centre shift <= 1e-4 * mean(var(X, axis=0)), or 300 iterations);
  - an empty cluster keeps its centre (sklearn relocates it);
  - the points are the fp32 embeddings (Inception features are fp32; the reference's float64 copy of them is exact);
  - `random_state` (default None: NumPy's global state, as sklearn's None means) draws the seeding uniforms."""
import numpy as np

from . import eval_task

_N_INIT = 10
_MAX_ITER = 300


def compute_prd(eval_dist, ref_dist, num_angles=1001, epsilon=1e-10):
  """PRD curve of two discrete distributions (reference prd_score.py:42-91): for each slope lambda = tan(angle) on an
  equiangular grid of num_angles angles in [epsilon, pi/2 - epsilon], precision = sum_i min(lambda ref_i, eval_i) and
  recall = precision / lambda.  Returns (precision, recall), each [num_angles]."""
  if not 0 < epsilon < 0.1:
    raise ValueError("epsilon must lie in (0, 0.1), got %s." % str(epsilon))
  if not 3 <= num_angles <= 1e6:
    raise ValueError("num_angles must lie in [3, 1e6], got %s." % str(num_angles))
  lam = np.tan(np.linspace(epsilon, np.pi / 2 - epsilon, num=num_angles))
  ev, rf = np.asarray(eval_dist)[None, :], np.asarray(ref_dist)[None, :]
  precision = np.sum(np.minimum(lam[:, None] * rf, ev), axis=1)
  return precision, precision / lam


def _random_state(random_state):
  if random_state is None:
    return np.random.mtrand._rand
  if isinstance(random_state, np.random.RandomState):
    return random_state
  return np.random.RandomState(random_state)


def _densities(counts):
  """np.histogram(labels, bins=k, range=[0, k], density=True) from the per-cluster counts (unit-width bins)."""
  counts = np.asarray(counts, np.int64)
  return counts / np.ones(len(counts)) / counts.sum()


def _cluster_runs(eval_data, ref_data, num_clusters, num_runs, random_state):
  """Clusters the union of both sets num_runs times on the device.  Returns the per-run cluster counts
  [num_runs, 2, num_clusters] (eval rows, ref rows) and the Lloyd iterations per run."""
  import torch
  from .. import kernels as K
  x_host = np.vstack([np.asarray(eval_data, np.float32).reshape(len(eval_data), -1),
                      np.asarray(ref_data, np.float32).reshape(len(ref_data), -1)])
  m = len(x_host)
  uniforms = _random_state(random_state).random_sample((num_runs * _N_INIT, num_clusters))
  tol = 1e-4 * np.mean(np.var(x_host.astype(np.float64), axis=0))
  x = torch.from_numpy(x_host).to(K._RT["device"])
  seeds = K.kmeans_seed(x, uniforms)
  _, inertia, _ = K.kmeans_finish(x, seeds, len(eval_data))
  best = np.argmin(inertia.reshape(num_runs, _N_INIT), axis=1) + _N_INIT * np.arange(num_runs)
  centroids = seeds[torch.from_numpy(best).to(seeds.device)].contiguous()
  labels = torch.empty(num_runs, m, dtype=torch.int32, device=x.device)
  state = torch.zeros(num_runs, 2, dtype=torch.int32, device=x.device)
  for _ in range(_MAX_ITER):
    K.kmeans_lloyd_step(x, centroids, labels, state, tol)
    st = state.cpu().numpy()
    if (st[:, 0] != 0).all():
      break
  _, _, counts = K.kmeans_finish(x, centroids, len(eval_data))
  return counts, st[:, 1]


def _cluster_into_bins(eval_data, ref_data, num_clusters, random_state=None):
  """Clusters the union of the data points; returns the histograms (densities over the clusters) of eval_data and
  ref_data (reference prd_score.py:94-122)."""
  counts, _ = _cluster_runs(eval_data, ref_data, num_clusters, 1, random_state)
  return _densities(counts[0, 0]), _densities(counts[0, 1])


def compute_prd_from_embedding(eval_data, ref_data, num_clusters=20, num_angles=1001, num_runs=10,
                               enforce_balance=True, random_state=None):
  """PRD curve of two embeddings, averaged over num_runs clusterings (reference prd_score.py:125-177).
  Returns (precision, recall), each [num_angles]."""
  if enforce_balance and len(eval_data) != len(ref_data):
    raise ValueError("eval_data has %d points and ref_data %d: unbalanced sets bias the clustering towards the larger "
                     "one (pass enforce_balance=False to allow it)" % (len(eval_data), len(ref_data)))
  counts, _ = _cluster_runs(eval_data, ref_data, num_clusters, num_runs, random_state)
  precisions, recalls = [], []
  for r in range(num_runs):
    precision, recall = compute_prd(_densities(counts[r, 0]), _densities(counts[r, 1]), num_angles)
    precisions.append(precision)
    recalls.append(recall)
  return np.mean(precisions, axis=0), np.mean(recalls, axis=0)


def _check_prd(precision, recall, beta):
  for name, v in (("precision", precision), ("recall", recall)):
    if not np.all((v >= 0) & (v <= 1)):
      raise ValueError("every %s value must lie in [0, 1]." % name)
  if beta <= 0:
    raise ValueError("beta must be positive, got %s." % str(beta))


def _prd_to_f_beta(precision, recall, beta=1, epsilon=1e-10):
  """F_beta = (1 + beta^2) p r / (beta^2 p + r + epsilon) of every (p, r) pair (reference prd_score.py:180-213)."""
  _check_prd(precision, recall, beta)
  b2 = beta ** 2
  return (1 + b2) * (precision * recall) / (b2 * precision + recall + epsilon)


def prd_to_max_f_beta_pair(precision, recall, beta=8):
  """(max F_beta, max F_{1/beta}) over a PRD curve: one number that tracks recall and one that tracks precision
  (reference prd_score.py:216-248)."""
  precision, recall = np.asarray(precision), np.asarray(recall)
  _check_prd(precision, recall, beta)
  return np.max(_prd_to_f_beta(precision, recall, beta)), np.max(_prd_to_f_beta(precision, recall, 1 / beta))


def plot(precision_recall_pairs, labels=None, out_path=None, legend_loc="lower left", dpi=150):
  """Draws recall (x) against precision (y) for each (precision, recall) pair and saves the figure to out_path, or shows
  it when out_path is None (reference prd_score.py:251-299).  matplotlib is imported only once the arguments are valid."""
  if labels is not None and len(labels) != len(precision_recall_pairs):
    raise ValueError("got %d labels for %d precision/recall pairs." % (len(labels), len(precision_recall_pairs)))
  import matplotlib.pyplot as plt
  fig, ax = plt.subplots(figsize=(3.5, 3.5), dpi=dpi)
  ax.tick_params(axis="both", which="major", labelsize=12)
  for i, (precision, recall) in enumerate(precision_recall_pairs):
    ax.plot(recall, precision, label=None if labels is None else labels[i], alpha=0.5, linewidth=3)
  if labels is not None:
    ax.legend(loc=legend_loc)
  ax.set_xlim(0, 1)
  ax.set_ylim(0, 1)
  ax.set_xlabel("Recall", fontsize=12)
  ax.set_ylabel("Precision", fontsize=12)
  fig.tight_layout()
  if out_path is None:
    plt.show()
  else:
    fig.savefig(out_path, bbox_inches="tight", dpi=dpi)
    plt.close(fig)


class PRDScoreTask(eval_task.EvalTask):
  """max F_8 (tracks recall) and max F_1/8 (tracks precision) of the PRD curve of the generated against the real
  Inception pool_3 features, with a fixed seed.  Needs the features (keep_features=True).  In a sharded evaluation every
  rank holds all gathered features and computes the same value."""
  _LABEL = "prd"

  def __init__(self, num_clusters=20, num_angles=1001, num_runs=10, seed=0):
    self.num_clusters, self.num_angles, self.num_runs, self.seed = num_clusters, num_angles, num_runs, seed

  def metric_list(self):
    return frozenset(["prd_f8", "prd_f1_8"])

  def run_after_session(self, fake_dset, real_dset):
    if fake_dset.activations is None or real_dset.activations is None:
      raise ValueError("PRDScoreTask needs the Inception features of both sets: evaluate with keep_features=True")
    precision, recall = compute_prd_from_embedding(fake_dset.activations, real_dset.activations, self.num_clusters,
                                                   self.num_angles, self.num_runs, random_state=self.seed)
    # the density histograms may sum to 1 + 1 ulp, which puts recall at small slopes one ulp above 1
    f_beta, f_beta_inv = prd_to_max_f_beta_pair(np.clip(precision, 0, 1), np.clip(recall, 0, 1), beta=8)
    return {"prd_f8": float(f_beta), "prd_f1_8": float(f_beta_inv)}
