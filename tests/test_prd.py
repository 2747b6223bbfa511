"""PRD precision / recall (reference metrics/prd_score.py): the reference's own cases restated, the float64 clustering
oracle (tests/prd_oracle.py) against sklearn's Lloyd, a closed-form mixture, agreement with the reference's
MiniBatchKMeans formulation, the device k-means entries (csrc/kmeans.cu) against the oracle, their determinism and
argument errors, and the metric inside the evaluation loop."""
import os

import numpy as np
import pytest

from tests import prd_oracle as oracle
from tests.abi_emulator import EmulatedLib, emulated_library, f32, f64, i32


def _prd():
  from compare_gan_b200.metrics import prd_score
  return prd_score


def _mixture(rs, n, d, centers, weights=None, noise=1.0):
  """n fp32 points around the given centres (mode i drawn with probability weights[i])."""
  idx = rs.choice(len(centers), size=n, p=weights)
  return (centers[idx] + noise * rs.randn(n, d)).astype(np.float32)


# ---- 1. the reference's PRD cases (prd_score_test.py), restated ----

def test_compute_prd_values():
  prd = _prd()
  assert np.allclose(np.ravel(prd.compute_prd([0, 1], [1, 0])), 0, atol=1e-7)
  p, r = prd.compute_prd([1, 0], [1, 0], num_angles=11)
  assert np.allclose([p[5], r[5]], [1, 1], atol=1e-7)
  p, r = prd.compute_prd([0.5, 0.5], [1, 0], num_angles=11)
  assert np.allclose([p[5], r[5], p[10], r[1]], [0.5, 0.5, 0.5, 1], atol=1e-7)
  p, r = prd.compute_prd([1, 0], [0.5, 0.5], num_angles=11)
  assert np.allclose([p[5], r[5], r[1], p[10]], [0.5, 0.5, 0.5, 1], atol=1e-7)
  want = oracle.compute_prd(np.array([0.2, 0.3, 0.5]), np.array([0.6, 0.1, 0.3]), 101)
  got = prd.compute_prd(np.array([0.2, 0.3, 0.5]), np.array([0.6, 0.1, 0.3]), 101)
  assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


@pytest.mark.parametrize("kw", [dict(epsilon=0), dict(epsilon=1), dict(epsilon=-1), dict(num_angles=0),
                                dict(num_angles=1), dict(num_angles=-1), dict(num_angles=1e6 + 1), dict(num_angles=2.5)])
def test_compute_prd_argument_errors(kw):
  with pytest.raises(ValueError):
    _prd().compute_prd([1], [1], **kw)


def test_prd_to_f_beta_values_and_errors():
  prd = _prd()
  p = np.array([1, 1, 0, 0, 0.5, 1, 0.5])
  r = np.array([1, 0, 1, 0, 0.5, 0.5, 1])
  for beta, want in [(1, [1, 0, 0, 0, 0.5, 2 / 3, 2 / 3]), (2, [1, 0, 0, 0, 0.5, 5 / 9, 5 / 6]),
                     (0.5, [1, 0, 0, 0, 0.5, 5 / 6, 5 / 9])]:
    with np.errstate(invalid="ignore"):
      assert np.allclose(prd._prd_to_f_beta(p, r, beta=beta), want, atol=1e-7), beta
  assert prd._prd_to_f_beta(np.array([]), np.array([]), beta=1).shape == (0,)
  for args, beta in [((np.ones(1), np.ones(1)), 0), ((np.ones(1), np.ones(1)), -3), ((-np.ones(1), np.ones(1)), 1),
                     ((np.ones(1), -np.ones(1)), 1)]:
    with pytest.raises(ValueError):
      prd._prd_to_f_beta(*args, beta=beta)
  with pytest.raises(ValueError):
    prd.prd_to_max_f_beta_pair(np.ones(3), 2 * np.ones(3))
  assert prd.prd_to_max_f_beta_pair(np.ones(3), np.ones(3)) == pytest.approx((1.0, 1.0), abs=1e-9)


@pytest.mark.parametrize("pairs,labels", [(np.zeros([3, 2, 5]), ["1", "2"]), (np.zeros([1, 2, 5]), ["1", "2", "3"])])
def test_plot_label_count_error(pairs, labels):
  with pytest.raises(ValueError):       # raised before matplotlib is imported
    _prd().plot(pairs, labels=labels)


# ---- the device entries, emulated on the CPU through the oracle ----

def _emulated_seed(self, c, x, m, d, k, groups, uni):
  xs = f32(x, m * d).reshape(m, d).astype(np.float64)
  u = f64(uni, groups * k).reshape(groups, k)
  assert k <= m and ((u >= 0) & (u < 1)).all()
  f64(c, groups * k * d)[:] = np.concatenate([oracle.seed(xs, u[g]).ravel() for g in range(groups)])


def _emulated_lloyd_step(self, c, labels, state, x, m, d, k, groups, tol):
  xs = f32(x, m * d).reshape(m, d).astype(np.float64)
  cs = f64(c, groups * k * d).reshape(groups, k, d)
  lab = i32(labels, groups * m).reshape(groups, m)
  st = i32(state, groups * 2).reshape(groups, 2)
  for g in range(groups):
    oracle.lloyd_step(xs, cs[g], lab[g], st[g], tol)


def _emulated_finish(self, labels, inertia, counts, c, x, m, d, k, groups, n_eval):
  xs = f32(x, m * d).reshape(m, d).astype(np.float64)
  cs = f64(c, groups * k * d).reshape(groups, k, d)
  for g in range(groups):
    lab, dist = oracle.assign(xs, cs[g])
    i32(labels, groups * m)[g * m:(g + 1) * m] = lab
    f64(inertia, groups)[g] = dist.sum()
    i32(counts, groups * 2 * k)[g * 2 * k:(g + 1) * 2 * k] = np.concatenate(
        [np.bincount(lab[:n_eval], minlength=k), np.bincount(lab[n_eval:], minlength=k)])


def _patch(setattr_fn):
  setattr_fn(EmulatedLib, "cgan_kmeans_seed", _emulated_seed, raising=False)
  setattr_fn(EmulatedLib, "cgan_kmeans_lloyd_step", _emulated_lloyd_step, raising=False)
  setattr_fn(EmulatedLib, "cgan_kmeans_finish", _emulated_finish, raising=False)


@pytest.fixture
def emulated(monkeypatch):
  _patch(monkeypatch.setattr)
  from compare_gan_b200 import kernels as K
  with emulated_library():
    yield K


@pytest.fixture(scope="module")
def gpu():
  from compare_gan_b200 import kernels as K
  K.init(0)
  return K


def test_cluster_into_bins_with_an_empty_cluster(emulated):
  ev, rf = _prd()._cluster_into_bins(np.zeros([5, 4]), np.ones([5, 4]), 3, random_state=0)
  assert len(ev) == len(rf) == 3
  assert abs(ev.sum() - 1) < 1e-12 and abs(rf.sum() - 1) < 1e-12
  assert sorted(ev) == [0, 0, 1] and sorted(rf) == [0, 0, 1]     # two distinct points: one cluster stays empty


def test_enforce_balance(emulated):
  prd = _prd()
  with pytest.raises(ValueError):
    prd.compute_prd_from_embedding(np.array([[0], [0], [1]]), np.array([[0], [1]]), num_clusters=2, enforce_balance=True)
  p, r = prd.compute_prd_from_embedding(np.array([[0], [0], [1]]), np.array([[0], [1]]), num_clusters=2,
                                        enforce_balance=False, random_state=1)
  assert p.shape == r.shape == (1001,)


# ---- 2. the oracle's Lloyd against sklearn ----

@pytest.mark.parametrize("spread", [0.3, 1.0, 6.0])
def test_oracle_lloyd_matches_sklearn(spread):
  sk = pytest.importorskip("sklearn.cluster")
  rs = np.random.RandomState(int(spread * 10))
  x = np.abs(_mixture(rs, 4000, 64, rs.rand(20, 64) * spread, noise=0.5)).astype(np.float64)
  c0 = oracle.seed(x, rs.random_sample(20))
  lab, inertia, c, it = oracle.lloyd(x, c0, oracle.tolerance(x))
  km = sk.KMeans(20, init=c0, n_init=1, algorithm="lloyd", tol=1e-4, max_iter=300).fit(x)
  assert np.array_equal(lab, km.labels_) and it == km.n_iter_, (it, km.n_iter_)
  assert abs(inertia - km.inertia_) <= 1e-12 * km.inertia_
  assert np.abs(c - km.cluster_centers_).max() <= 1e-12 * np.abs(c).max()
  assert it > 3


# ---- 3. a closed form: 20 separated modes, the eval set covering 10 of them uniformly ----

def test_closed_form_mode_dropping(emulated):
  rs = np.random.RandomState(3)
  centers = rs.randn(20, 40) * 100.0
  ref = (centers[np.repeat(np.arange(20), 100)] + 0.1 * rs.randn(2000, 40)).astype(np.float32)
  ev = (centers[np.repeat(np.arange(10), 200)] + 0.1 * rs.randn(2000, 40)).astype(np.float32)
  f8, f18 = oracle.max_f_beta_pair(*_prd().compute_prd_from_embedding(ev, ref, random_state=0))
  # every clustering finds the 20 modes: eval = 10 bins of 1/10, ref = 20 bins of 1/20, so at slope lambda
  # precision = min(lambda / 2, 1) and recall = min(1 / 2, 1 / lambda)
  lam = np.tan(np.linspace(1e-10, np.pi / 2 - 1e-10, 1001))
  prec = np.minimum(lam / 2, 1.0)
  want = oracle.max_f_beta_pair(prec, np.minimum(0.5, 1 / lam))
  assert abs(f8 - want[0]) <= 1e-9 and abs(f18 - want[1]) <= 1e-9, (f8, f18, want)


# ---- 4. agreement with the reference's formulation (sklearn MiniBatchKMeans, num_runs = 10) ----

def _reference_f_beta(ev, ref, seed, sk):
  x = np.vstack([ev, ref]).astype(np.float64)
  rs = np.random.RandomState(seed)
  curves = []
  for _ in range(10):
    lab = sk.MiniBatchKMeans(n_clusters=20, n_init=10, random_state=rs).fit(x).labels_
    he = np.histogram(lab[:len(ev)], bins=20, range=[0, 20], density=True)[0]
    hr = np.histogram(lab[len(ev):], bins=20, range=[0, 20], density=True)[0]
    curves.append(oracle.compute_prd(he, hr))
  return oracle.max_f_beta_pair(np.mean([c[0] for c in curves], 0), np.mean([c[1] for c in curves], 0))


# The reference formulation's spread over 10 seeds, measured with this test's data (the modes are well separated, so
# every fit finds them): mode dropping sigma(F8) = 6e-17, sigma(F1/8) = 2e-16; mode collapsing sigma = 0 for both.
# The bound is therefore max(0.02, 3 sigma) = 0.02.
@pytest.mark.parametrize("case", ["dropping", "collapsing"])
def test_agrees_with_the_reference_formulation(emulated, case):
  sk = pytest.importorskip("sklearn.cluster")
  rs = np.random.RandomState(11)
  centers = rs.randn(20, 16) * 10.0
  ref = _mixture(rs, 1000, 16, centers)
  if case == "dropping":
    ev = _mixture(rs, 1000, 16, centers[:12])
  else:
    w = np.full(20, 0.5 / 19)
    w[0] = 0.5
    ev = _mixture(rs, 1000, 16, centers, weights=w)
  refs = np.array([_reference_f_beta(ev, ref, s, sk) for s in range(10)])
  sigma = refs.std(axis=0)
  p, r = _prd().compute_prd_from_embedding(ev, ref, random_state=0)
  got = oracle.max_f_beta_pair(p, r)
  tol = np.maximum(0.02, 3 * sigma)
  assert (np.abs(np.array(got) - refs.mean(axis=0)) <= tol).all(), (got, refs.mean(axis=0), sigma)
  assert sigma.max() < 0.02, sigma


# ---- 5. the host code above the emulator ----

def test_task_keys_and_missing_features():
  from compare_gan_b200 import eval_utils
  prd = _prd()
  task = prd.PRDScoreTask()
  assert task.metric_list() == frozenset(["prd_f8", "prd_f1_8"]) and task.images_needed == 0
  fake, real = eval_utils.EvalDataSample(), eval_utils.EvalDataSample()
  with pytest.raises(ValueError, match="keep_features"):
    task.run_after_session(fake, real)


def check_evaluation(K, use_graph):
  """evaluate() with PRD next to FID / IS: the score equals the oracle on the evaluation's own features, the graph path
  equals the eager one, and FID / IS are bit-identical to a run without the PRD task."""
  from compare_gan_b200 import eval_gan_lib
  from compare_gan_b200.metrics import fid_score, inception_score
  from tests.gpu_util import make_pair
  prd = _prd()
  seen = []

  class Recorder(prd.PRDScoreTask):
    def run_after_session(self, fake_dset, real_dset):
      seen.append((fake_dset.activations, real_dset.activations))
      return super(Recorder, self).run_after_session(fake_dset, real_dset)
  eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True)
  base = [fid_score.FIDScoreTask(), inception_score.InceptionScoreTask()]
  n = 144 if use_graph else 64
  real = np.random.RandomState(5).rand(n, 32, 32, 3).astype(np.float32)
  kw = dict(num_averaging_runs=1, num_samples=n, batch_size=32, seed=7, real_images=real)
  res = eval_gan_lib.evaluate(eng, base + [Recorder(num_runs=2)], use_graph=use_graph, **kw)
  without = eval_gan_lib.evaluate(eng, base, use_graph=use_graph, **kw)
  for key in ("fid_score_mean", "inception_score_mean"):
    assert res[key] == without[key], key
  if use_graph:
    eager = eval_gan_lib.evaluate(eng, base + [prd.PRDScoreTask(num_runs=2)], use_graph=False, **kw)
    assert res["prd_f8_mean"] == eager["prd_f8_mean"] and res["prd_f1_8_mean"] == eager["prd_f1_8_mean"]
  fake_acts, real_acts = seen[0]
  u = np.random.RandomState(0).random_sample((2 * 10, 20))
  p, r, _ = oracle.prd_from_embedding(fake_acts, real_acts, u, num_runs=2)
  want = oracle.max_f_beta_pair(np.clip(p, 0, 1), np.clip(r, 0, 1))
  assert abs(res["prd_f8_mean"] - want[0]) <= 1e-12 and abs(res["prd_f1_8_mean"] - want[1]) <= 1e-12, (res, want)


def test_evaluation_with_prd_on_the_emulator(emulated):
  check_evaluation(emulated, use_graph=False)


def _rank_worker(rank, world, port, q):
  import torch.distributed as dist
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  _patch(lambda obj, name, fn, raising=False: setattr(obj, name, fn))
  from compare_gan_b200 import eval_utils
  from compare_gan_b200.metrics import prd_score
  with emulated_library():
    from compare_gan_b200 import kernels as K
    rs = np.random.RandomState(20 + rank)           # every rank generates different samples
    centers = np.random.RandomState(1).randn(20, 16) * 4
    samples = []
    for which in range(2):
      acc = eval_utils.FeatureAccumulator(dim=16)
      pool = _mixture(rs, 40, 16, centers[:10] if which == 0 else centers)
      acc.add(K.from_numpy(pool), K.from_numpy(np.zeros((40, 8), np.float32)), 40)
      samples.append(acc.finish(eval_utils.EvalDataSample()))
    got = prd_score.PRDScoreTask(num_runs=2).run_after_session(samples[0], samples[1])
  q.put((rank, got, samples[0].activations.shape[0]))
  dist.barrier()
  dist.destroy_process_group()


def test_two_rank_score_is_the_same_on_both_ranks():
  import socket
  import torch.multiprocessing as mp
  s = socket.socket()
  s.bind(("127.0.0.1", 0))
  port = s.getsockname()[1]
  s.close()
  ctx = mp.get_context("spawn")
  q = ctx.Queue()
  procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, q)) for r in range(2)]
  for p in procs:
    p.start()
  res = dict((r, (g, n)) for r, g, n in (q.get(timeout=300) for _ in procs))
  for p in procs:
    p.join(60)
    assert p.exitcode == 0
  assert res[0][1] == res[1][1] == 80          # the gathered features of both ranks
  assert res[0][0] == res[1][0]


# ---- 6.-9. the device entries ----

SHAPES = [(5, 1, 2, 10), (10, 4, 3, 1), (1999, 37, 7, 3), (2000, 2048, 20, 100), (20000, 2048, 20, 10)]


def _data(m, d, k, seed=0):
  rs = np.random.RandomState(seed)
  centers = rs.randn(2 * k, d)                # more modes than clusters: clusters merge modes, Lloyd has work to do
  x = np.abs(_mixture(rs, m, d, centers, noise=0.5))
  return x, rs


def _run_lloyd(K, xd, c, max_iter=oracle.MAX_ITER):
  import torch
  groups, _, _ = c.shape
  m = xd.shape[0]
  labels = torch.empty(groups, m, dtype=torch.int32, device=xd.device)
  state = torch.zeros(groups, 2, dtype=torch.int32, device=xd.device)
  tol = oracle.tolerance(xd.cpu().numpy().astype(np.float64))
  for _ in range(max_iter):
    K.kmeans_lloyd_step(xd, c, labels, state, tol)
    if (state.cpu().numpy()[:, 0] != 0).all():
      break
  return state.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_entries_match_the_oracle(gpu, shape):
  import torch
  m, d, k, groups = shape
  x, rs = _data(m, d, k, seed=m + d)
  x64 = x.astype(np.float64)
  u = rs.random_sample((groups, k))
  xd = torch.from_numpy(x).cuda()
  c0 = gpu.kmeans_seed(xd, u)
  want0 = np.stack([oracle.seed(x64, u[g]) for g in range(groups)])
  assert np.array_equal(c0.cpu().numpy(), want0)
  _, inertia0, counts0 = gpu.kmeans_finish(xd, c0, m // 2)
  for g in range(groups):
    lab, dist = oracle.assign(x64, want0[g])
    assert np.array_equal(counts0[g], [np.bincount(lab[:m // 2], minlength=k), np.bincount(lab[m // 2:], minlength=k)])
    assert abs(inertia0[g] - dist.sum()) <= 1e-12 * dist.sum()
  c = c0.clone()
  state = _run_lloyd(gpu, xd, c)
  labels, inertia, counts = gpu.kmeans_finish(xd, c, m // 2)
  labels = labels.cpu().numpy()
  tol = oracle.tolerance(x64)
  cs = c.cpu().numpy()
  for g in range(groups):
    lab, inert, cg, it = oracle.lloyd(x64, want0[g], tol)
    assert state[g, 1] == it, (g, state[g], it)
    assert np.array_equal(labels[g], lab), g
    assert np.array_equal(counts[g], [np.bincount(lab[:m // 2], minlength=k), np.bincount(lab[m // 2:], minlength=k)])
    assert abs(inertia[g] - inert) <= 1e-12 * max(inert, 1e-300), (inertia[g], inert)
    assert np.abs(cs[g] - cg).max() <= 1e-12 * max(np.abs(cg).max(), 1e-300)


@pytest.mark.gpu
def test_determinism_and_degenerate_sets(gpu):
  import torch
  x, rs = _data(3000, 200, 20, seed=9)
  xd = torch.from_numpy(x).cuda()
  u = rs.random_sample((12, 20))
  u[7] = u[2]                                          # identical uniforms: identical groups

  def full(uu):
    c = gpu.kmeans_seed(xd, uu)
    st = _run_lloyd(gpu, xd, c)
    lab, inert, cnt = gpu.kmeans_finish(xd, c, 1500)
    return c.cpu().numpy(), st, lab.cpu().numpy(), inert, cnt
  a, b = full(u), full(u)
  for p, q in zip(a, b):
    assert np.array_equal(p, q)                       # reruns are bit-identical
  alone = full(u[5:6])
  for p, q in zip(a, alone):
    assert np.array_equal(p[5], q[0])                 # a group alone equals the same group in the batch
  for p in a:
    assert np.array_equal(p[7], p[2])
  for pts in (np.repeat(x[:3], 40, axis=0), np.ones((50, 7), np.float32), x[:20]):   # duplicates, identical, m == k
    pd = torch.from_numpy(np.ascontiguousarray(pts)).cuda()
    c = gpu.kmeans_seed(pd, rs.random_sample((3, 20)))
    st = _run_lloyd(gpu, pd, c)
    lab, inert, cnt = gpu.kmeans_finish(pd, c, len(pts) // 2)
    assert (st[:, 0] != 0).all() and cnt.sum() == 3 * len(pts) and np.isfinite(inert).all()
  torch.cuda.synchronize()


@pytest.mark.gpu
def test_argument_errors(gpu):
  import torch
  lib = gpu.lib()
  x = torch.zeros(10, 4, device="cuda")
  c = torch.zeros(2, 3, 4, dtype=torch.float64, device="cuda")
  lab = torch.zeros(2, 10, dtype=torch.int32, device="cuda")
  st = torch.zeros(2, 2, dtype=torch.int32, device="cuda")
  inert = torch.zeros(2, dtype=torch.float64, device="cuda")
  cnt = torch.zeros(2, 2, 3, dtype=torch.int32, device="cuda")
  u = np.full((2, 3), 0.5)
  X, C, L, S, I, N = x.data_ptr(), c.data_ptr(), lab.data_ptr(), st.data_ptr(), inert.data_ptr(), cnt.data_ptr()
  shapes = [dict(m=2), dict(k=0), dict(d=0), dict(groups=0), dict(k=65, m=100)]
  cases = {
      "cgan_kmeans_seed": ([dict(c=None), dict(x=None), dict(u=None), dict(u=np.full((2, 3), 1.0)),
                            dict(u=np.full((2, 3), -0.1)), dict(u=np.full((2, 3), np.nan))] + shapes,
                           lambda a: (a["c"], a["x"], a["m"], a["d"], a["k"], a["groups"],
                                      None if a["u"] is None else a["u"].ctypes.data)),
      "cgan_kmeans_lloyd_step": ([dict(c=None), dict(lab=None), dict(st=None), dict(x=None), dict(tol=-1.0)] + shapes,
                                 lambda a: (a["c"], a["lab"], a["st"], a["x"], a["m"], a["d"], a["k"], a["groups"],
                                            a["tol"])),
      "cgan_kmeans_finish": ([dict(lab=None), dict(inert=None), dict(cnt=None), dict(c=None), dict(x=None),
                              dict(n_eval=-1), dict(n_eval=11)] + shapes,
                             lambda a: (a["lab"], a["inert"], a["cnt"], a["c"], a["x"], a["m"], a["d"], a["k"],
                                        a["groups"], a["n_eval"])),
  }
  for name, (bad, args) in cases.items():
    fn = lib.fn[name]
    for case in bad:
      a = dict(c=C, x=X, lab=L, st=S, inert=I, cnt=N, u=u, m=10, d=4, k=3, groups=2, tol=0.0, n_eval=5)
      a.update(case)
      assert fn(lib.ctx, *args(a)) == 1, (name, case)
      assert lib.fn["cgan_last_error"](lib.ctx).decode().startswith(name + ":"), (name, case)
  c = gpu.kmeans_seed(x, u)                             # the context is still usable
  gpu.kmeans_finish(x, c, 5)
  torch.cuda.synchronize()


@pytest.mark.gpu
def test_end_to_end_at_cifar_size(gpu):
  rs = np.random.RandomState(4)
  centers = rs.randn(30, 2048) * 0.2
  ref = np.abs(_mixture(rs, 10000, 2048, centers, noise=0.5))
  ev = np.abs(_mixture(rs, 10000, 2048, centers[:18], noise=0.5))
  prd = _prd()
  p, r = prd.compute_prd_from_embedding(ev, ref, random_state=123)
  u = np.random.RandomState(123).random_sample((100, 20))
  wp, wr, counts = oracle.prd_from_embedding(ev, ref, u)
  got_counts, _ = prd._cluster_runs(ev, ref, 20, 10, 123)
  assert np.array_equal(got_counts, counts)
  assert np.abs(p - wp).max() <= 1e-12 and np.abs(r - wr).max() <= 1e-12


@pytest.mark.gpu
def test_evaluation_with_prd(gpu):
  check_evaluation(gpu, use_graph=True)
