"""TEST INFRASTRUCTURE ONLY: a float64 NumPy restatement of the engine's PRD clustering (compare_gan_b200/metrics/
prd_score.py, csrc/kmeans.cu): k-means++ seeding from given uniforms, sklearn KMeans(algorithm="lloyd")'s loop with
empty clusters keeping their centre, best-of-n_init by inertia, and the reference's histograms and curves
(reference metrics/prd_score.py:42-177).  It also backs the emulated C-ABI entries of tests/test_prd.py."""
import numpy as np

MAX_ITER = 300


def sq_dist(x, c):
  """||x||^2 + ||c||^2 - 2 x.c: [m, k] float64, the device's expansion."""
  return (np.einsum("ij,ij->i", x, x)[:, None] + np.einsum("ij,ij->i", c, c)[None, :]) - 2.0 * (x @ c.T)


def assign(x, c):
  """Nearest centre (first minimum) and its squared distance."""
  d = sq_dist(x, c)
  lab = np.argmin(d, axis=1).astype(np.int32)
  return lab, d[np.arange(len(x)), lab]


def seed(x, u):
  """k-means++ from the uniforms u [k]: centre 0 is point min(floor(u0 m), m-1), centre j the smallest i with
  cumsum(w)[i] > u_j * cumsum(w)[-1] (w: squared distance to the nearest chosen centre, clamped at 0), or
  min(floor(u_j m), m-1) when that sum is 0."""
  m = len(x)
  idx = min(int(np.floor(u[0] * m)), m - 1)
  cs = [x[idx]]
  w = np.maximum(sq_dist(x, x[idx:idx + 1])[:, 0], 0.0)
  for j in range(1, len(u)):
    cum = np.cumsum(w)
    if cum[-1] > 0.0:
      hit = np.nonzero(cum > u[j] * cum[-1])[0]
      idx = int(hit[0]) if len(hit) else m - 1
    else:
      idx = min(int(np.floor(u[j] * m)), m - 1)
    cs.append(x[idx])
    w = np.minimum(w, np.maximum(sq_dist(x, x[idx:idx + 1])[:, 0], 0.0))
  return np.stack(cs)


def lloyd_step(x, c, labels, state, tol):
  """One Lloyd iteration of one group, in place: c [k, d], labels [m], state [2] = (status, iterations)."""
  if state[0] != 0:
    return
  lab, _ = assign(x, c)
  changed = state[1] == 0 or not np.array_equal(lab, labels)
  old = c.copy()
  member = lab[None, :] == np.arange(len(c))[:, None]
  cnt = member.sum(axis=1)
  sums = member.astype(np.float64) @ x
  full = cnt > 0                       # an empty cluster keeps its centre
  c[full] = sums[full] / cnt[full, None]
  labels[:] = lab
  state[1] += 1
  if not changed:
    state[0] = 2
  elif ((c - old) ** 2).sum() <= tol:
    state[0] = 1


def tolerance(x, tol=1e-4):
  return tol * np.mean(np.var(x, axis=0))


def lloyd(x, c0, tol, max_iter=MAX_ITER):
  """Lloyd from c0 until converged or max_iter, then the final assignment: (labels, inertia, centres, iterations)."""
  c = np.array(c0, np.float64, copy=True)
  labels = np.zeros(len(x), np.int32)
  state = np.zeros(2, np.int64)
  while state[0] == 0 and state[1] < max_iter:
    lloyd_step(x, c, labels, state, tol)
  lab, dist = assign(x, c)
  return lab, dist.sum(), c, int(state[1])


def cluster_runs(x, n_eval, uniforms, num_runs, n_init, max_iter=MAX_ITER):
  """Best of n_init seedings by inertia, one Lloyd run from it, per run: (labels [runs, m], counts [runs, 2, k],
  iterations [runs])."""
  x = np.asarray(x, np.float64)
  tol = tolerance(x)
  labels, counts, iters = [], [], []
  for r in range(num_runs):
    seeds = [seed(x, uniforms[r * n_init + s]) for s in range(n_init)]
    inertias = [assign(x, c)[1].sum() for c in seeds]
    lab, _, _, it = lloyd(x, seeds[int(np.argmin(inertias))], tol, max_iter)
    k = uniforms.shape[1]
    labels.append(lab)
    counts.append([np.bincount(lab[:n_eval], minlength=k), np.bincount(lab[n_eval:], minlength=k)])
    iters.append(it)
  return np.array(labels), np.array(counts, np.int64), np.array(iters)


def compute_prd(eval_dist, ref_dist, num_angles=1001, epsilon=1e-10):
  slopes = np.tan(np.linspace(epsilon, np.pi / 2 - epsilon, num=num_angles))
  precision = np.minimum(np.asarray(ref_dist)[None, :] * slopes[:, None], np.asarray(eval_dist)[None, :]).sum(axis=1)
  return precision, precision / slopes


def prd_from_embedding(eval_data, ref_data, uniforms, num_clusters=20, num_angles=1001, num_runs=10, n_init=10):
  """The engine's compute_prd_from_embedding given its uniforms [num_runs * n_init, num_clusters]; the points are the
  fp32 features the device reads.  Returns (precision, recall, counts)."""
  x = np.vstack([np.asarray(eval_data, np.float32), np.asarray(ref_data, np.float32)]).astype(np.float64)
  n = len(eval_data)
  _, counts, _ = cluster_runs(x, n, uniforms, num_runs, n_init)
  curves = []
  for r in range(num_runs):
    ev = np.histogram(np.repeat(np.arange(num_clusters), counts[r, 0]), bins=num_clusters, range=[0, num_clusters],
                      density=True)[0]
    rf = np.histogram(np.repeat(np.arange(num_clusters), counts[r, 1]), bins=num_clusters, range=[0, num_clusters],
                      density=True)[0]
    curves.append(compute_prd(ev, rf, num_angles))
  return np.mean([p for p, _ in curves], axis=0), np.mean([r for _, r in curves], axis=0), counts


def max_f_beta_pair(precision, recall, beta=8, epsilon=1e-10):
  def f(b):
    return (1 + b ** 2) * (precision * recall) / ((b ** 2 * precision) + recall + epsilon)
  return np.max(f(beta)), np.max(f(1.0 / beta))
