"""Fractal dimension (reference metrics/fractal_dimension.py): the reference's own cases restated on the numpy / scipy
restatement (tests/fractal_oracle.py), the host code above the emulated C-ABI, the device entries (csrc/fractal.cu)
against float64 cdist / np.less.outer, their row independence and argument errors, and the metric inside the
evaluation loop next to the reference test's other tasks."""
import ctypes
import os

import numpy as np
import pytest

from tests import fractal_oracle as oracle
from tests.abi_emulator import EmulatedLib, emulated_library, f32, f64


def _fd():
  from compare_gan_b200.metrics import fractal_dimension
  return fractal_dimension


def i64(ptr, n):
  return np.ctypeslib.as_array((ctypes.c_int64 * int(n)).from_address(int(ptr)))


# ---- the device entries, emulated on the CPU through the oracle ----

def _emulated_distances(self, out, x, n, seeds, s, d, scale):
  sc = np.float32(scale)
  xs = sc * f32(x, n * d).reshape(n, d)              # fp32(scale * v), as the device stages them
  ss = sc * f32(seeds, s * d).reshape(s, d)
  f64(out, n * s)[:] = oracle.distances(xs, ss).ravel()


def _emulated_range(self, out2, dist, count):
  v = f64(dist, count)
  nz = v[v > 0]
  f64(out2, 2)[:] = [nz.min() if len(nz) else np.inf, v.max()]


def _emulated_counts(self, counts, dist, count, edges, nedges):
  i64(counts, nedges)[:] = oracle.counts(f64(dist, count), f64(edges, nedges))


def _patch(setattr_fn):
  setattr_fn(EmulatedLib, "cgan_fd_distances", _emulated_distances, raising=False)
  setattr_fn(EmulatedLib, "cgan_fd_range", _emulated_range, raising=False)
  setattr_fn(EmulatedLib, "cgan_fd_counts", _emulated_counts, raising=False)


@pytest.fixture
def emulated(monkeypatch):
  _patch(monkeypatch.setattr)
  from tests.test_ms_ssim import _emulated_ssim_terms
  monkeypatch.setattr(EmulatedLib, "cgan_ssim_terms", _emulated_ssim_terms, raising=False)
  from compare_gan_b200 import kernels as K
  with emulated_library():
    yield K


@pytest.fixture(scope="module")
def gpu():
  from compare_gan_b200 import kernels as K
  K.init(0)
  return K


def _dev(K, a):
  import torch
  return torch.from_numpy(np.ascontiguousarray(a)).to(K._RT["device"])


# ---- 1. the reference's cases (fractal_dimension_test.py), restated with a seeded RNG ----

REFERENCE_CASES = [(1, 1.0, 0.05), (2, 2.0, 0.1)]


@pytest.mark.parametrize("dim,want,tol", REFERENCE_CASES)
def test_reference_cases_on_the_oracle(dim, want, tol):
  rs = np.random.RandomState(dim)
  x = rs.uniform(size=(10000, dim))
  got = oracle.fractal_dimension(x, rs.randint(10000, size=100))
  assert abs(got - want) <= tol, got


def check_reference_cases(K, dim, want, tol):
  x = np.random.RandomState(dim).uniform(size=(10000, dim)).astype(np.float32)
  got = _fd().compute_fractal_dimension(x, random_state=7)
  expect = oracle.fractal_dimension(x, np.random.RandomState(7).randint(10000, size=100))
  assert abs(got - want) <= tol, got
  return got, expect


@pytest.mark.parametrize("dim,want,tol", REFERENCE_CASES)
def test_reference_cases_on_the_emulator(emulated, dim, want, tol):
  got, expect = check_reference_cases(emulated, dim, want, tol)
  assert got == expect, (got, expect)


def test_global_random_state_draws_the_seeds_as_the_reference(emulated):
  x = np.random.RandomState(3).uniform(size=(500, 2)).astype(np.float32)
  np.random.seed(11)
  got = _fd().compute_fractal_dimension(x)
  np.random.seed(11)
  assert got == oracle.fractal_dimension(x, np.random.randint(500, size=100))


# ---- 2. the host tail and the count step ----

def test_host_tail_equals_the_oracle(emulated):
  rs = np.random.RandomState(4)
  pts = (rs.rand(3000, 6) @ rs.randn(6, 40)).astype(np.float32)
  dist = oracle.distances(pts, pts[:100])
  for n_bins, scale in [(1000, 0.1), (200, 0.2), (5000, 0.05)]:
    got = _fd().fractal_dimension_from_distances(_dev(emulated, dist), 3000, 100, n_bins, scale)
    assert got == oracle.slope_from_distances(dist, n_bins, scale), (n_bins, scale)


def _edge_cases():
  """Distances on edges, zeros and duplicates, and the edges themselves (with repeated edges)."""
  rs = np.random.RandomState(8)
  edges = np.sort(np.concatenate([rs.uniform(1, 100, 500), [5.0, 5.0, 7.25]]))
  dist = np.concatenate([edges[::3], edges[::3], np.zeros(37), rs.uniform(0, 120, 5000), [edges[0], edges[-1], 200.0],
                         np.nextafter(edges[::7], 0), np.nextafter(edges[::7], np.inf)])
  return rs.permutation(dist), edges


def check_counts_and_range(K):
  dist, edges = _edge_cases()
  d = _dev(K, dist)
  got = K.fd_counts(d, edges)
  assert got.dtype == np.int64 and np.array_equal(got, np.sum(np.less.outer(dist, edges), axis=0))
  lo, hi = K.fd_range(d)
  assert lo == np.min(dist[np.nonzero(dist)]) and hi == np.max(dist)
  lo, _ = K.fd_range(_dev(K, np.zeros(10)))
  assert lo == np.inf


def test_counts_and_range_on_the_emulator(emulated):
  check_counts_and_range(emulated)


# ---- 3. task and argument errors ----

def test_argument_and_task_errors(emulated):
  fd = _fd()
  x = np.random.RandomState(0).rand(50, 4).astype(np.float32)
  for bad in (x, np.zeros(200, np.float32)):            # 50 samples for 100 seeds; one axis only
    with pytest.raises(ValueError, match="N >= num_fd_seeds"):
      fd.compute_fractal_dimension(bad)
  with pytest.raises(ValueError, match="N >= num_fd_seeds"):
    fd.compute_fractal_dimension(x, num_fd_seeds=51)
  assert np.isfinite(fd.compute_fractal_dimension(x, num_fd_seeds=50, random_state=0))
  with pytest.raises(ValueError, match="identical"):
    fd.compute_fractal_dimension(np.ones((300, 3, 3, 1), np.float32), random_state=0)
  from compare_gan_b200 import eval_utils
  from compare_gan_b200.metrics import eval_task
  task = fd.FractalDimensionTask()
  assert task.metric_list() == frozenset(["fractal_dimension"])
  assert task.distance_seeds == 100 and task.images_needed >= 100
  small = fd.FractalDimensionTask(num_fd_seeds=16)
  assert small.distance_seeds == 16 and small.images_needed >= 16
  assert eval_task.EvalTask.distance_seeds == 0
  with pytest.raises(ValueError, match="N >= num_fd_seeds"):
    task.run_after_session(eval_utils.EvalDataSample(), None)           # fewer samples than seeds: no distances
  with pytest.raises(ValueError, match="identical"):
    task.run_after_session(eval_utils.EvalDataSample(seed_distances=_dev(emulated, np.zeros((300, 100)))), None)


# ---- 4. inside evaluate, with the reference test's task list ----

def check_evaluation(K, use_graph, conditional=False):
  """evaluate() with FID, fractal dimension, IS and MS-SSIM: the twelve keys, FID / IS bit-identical to a run without the
  new task, graph equal to eager, and the value equal to the oracle on the regenerated samples with seeds = the first
  S samples."""
  from compare_gan_b200 import eval_gan_lib
  from compare_gan_b200.metrics import fid_score, inception_score, ms_ssim_score
  from tests.gpu_util import make_pair
  fd = _fd()
  if conditional:
    # no spectral norm in G: its power iteration advances on every G call, so two evaluations would differ anyway
    eng, _ = make_pair("resnet_biggan_arch", (32, 32, 3), 4, loss="hinge", g_bn="conditional_batch_norm", d_sn=True,
                       conditional=True, num_classes=10, z_dim=120, ch=8)
  else:
    eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True)
  n, s = (300, 100) if use_graph else (64, 40)        # the seeds complete inside the second batch
  tasks = [fid_score.FIDScoreTask(), fd.FractalDimensionTask(num_fd_seeds=s), inception_score.InceptionScoreTask(),
           ms_ssim_score.MultiscaleSSIMTask(batch_size=16, num_batches=2)]
  base = [fid_score.FIDScoreTask(), inception_score.InceptionScoreTask()]
  real = np.random.RandomState(5).rand(n, 32, 32, 3).astype(np.float32)
  kw = dict(num_averaging_runs=1, num_samples=n, batch_size=32, seed=7, real_images=real)
  res = eval_gan_lib.evaluate(eng, tasks, use_graph=use_graph, **kw)
  for label in ("fid_score", "fractal_dimension", "inception_score", "ms_ssim"):
    for suffix in ("_mean", "_std", "_list"):
      assert label + suffix in res, label + suffix
  without = eval_gan_lib.evaluate(eng, base, use_graph=use_graph, **kw)
  for key in ("fid_score_mean", "inception_score_mean"):
    assert res[key] == without[key], key
  if use_graph:
    eager = eval_gan_lib.evaluate(eng, tasks, use_graph=False, **kw)
    assert res["fractal_dimension_mean"] == eager["fractal_dimension_mean"]
  rs = np.random.RandomState(7)
  imgs = np.concatenate([eval_gan_lib.generate_batch(eng, 32, rs).cpu() for _ in range((n + 31) // 32)])[:n]
  imgs = np.float32(255.0) * imgs.reshape(n, -1).astype(np.float32)
  want = oracle.fractal_dimension(imgs, np.arange(s))
  assert abs(res["fractal_dimension_mean"] - want) <= 1e-9 * max(1.0, abs(want)), (res["fractal_dimension_mean"], want)
  return res


def test_evaluation_on_the_emulator(emulated):
  check_evaluation(emulated, use_graph=False)


# ---- 5. sharded evaluation: rank 0's value, broadcast ----

def _rank_worker(rank, world, port, q):
  import torch.distributed as dist
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  _patch(lambda obj, name, fn, raising=False: setattr(obj, name, fn))
  from compare_gan_b200 import eval_utils
  from compare_gan_b200.metrics import fractal_dimension
  with emulated_library():
    from compare_gan_b200 import kernels as K
    x = np.random.RandomState(30 + rank).uniform(size=(400 + 50 * rank, 3)).astype(np.float32)   # rank-distinct samples
    xd = K.from_numpy(x).t
    dist_ = K.fd_distances(xd, xd[:20].contiguous(), 255.0)
    sample = eval_utils.EvalDataSample(seed_distances=dist_)
    got = fractal_dimension.FractalDimensionTask(num_fd_seeds=20).run_after_session(sample, None)["fractal_dimension"]
    local = fractal_dimension.fractal_dimension_from_distances(dist_, len(x), 20)
  q.put((rank, got, local))
  dist.barrier()
  dist.destroy_process_group()


def test_two_rank_score_is_rank_zeros():
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
  res = dict((r, (g, l)) for r, g, l in (q.get(timeout=300) for _ in procs))
  for p in procs:
    p.join(60)
    assert p.exitcode == 0
  assert res[0][0] == res[1][0] == res[0][1] and res[0][1] != res[1][1]


# ---- 6. the device entries ----

# (N, S, D): the reference's D = 1 and 2, image sizes up to 128^2 x 3, one and several seed tiles, N = 1 and N off the
# 64-row tile, and the CIFAR-size table
DIST_SHAPES = [(500, 100, 1), (777, 100, 2), (130, 100, 3072), (65, 130, 4320), (1, 1, 12288), (200, 100, 49152),
               (129, 1, 3072), (10000, 100, 3072)]


def _images(rs, n, d):
  """fp32 values in [0, 1] with near-duplicates: pairs of rows that differ in a single pixel by one step of 1/255."""
  x = rs.uniform(size=(n, d)).astype(np.float32)
  if n >= 8:
    x[n // 2] = x[1]
    x[n // 2, d // 2] = np.float32(min(1.0, x[1, d // 2] + 1 / 255.0))
  return x


@pytest.mark.gpu
@pytest.mark.parametrize("shape", DIST_SHAPES)
def test_distances_match_float64_cdist(gpu, shape):
  n, s, d = shape
  rs = np.random.RandomState(n + s + d)
  x = _images(rs, n, d)
  idx = rs.randint(n, size=s)
  idx[0] = n // 2 if n >= 8 else 0
  got = gpu.fd_distances(_dev(gpu, x), _dev(gpu, x[idx]), 255.0).cpu().numpy()
  x255 = np.float32(255.0) * x
  want = oracle.distances(x255, x255[idx])
  assert got.shape == (n, s)
  assert (np.abs(got - want) <= 1e-12 * want).all(), np.max(np.abs(got - want) / np.maximum(want, 1e-300))
  assert (got[idx, np.arange(s)] == 0).all()                    # every seed is at distance exactly 0 from itself
  assert ((got == 0) == (want == 0)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("d", [3072, 49152])
def test_rows_do_not_depend_on_the_call(gpu, d):
  import torch
  g = torch.Generator(device="cuda").manual_seed(d)
  n = 4000 if d > 40000 else 1000     # at 128^2 x 3 a call of 4000 rows runs in two row chunks
  x = torch.rand(n, d, device="cuda", generator=g)
  seeds = x[torch.arange(0, 200, 2, device="cuda")].contiguous()
  full = gpu.fd_distances(x, seeds, 255.0)
  assert torch.equal(full, gpu.fd_distances(x, seeds, 255.0))                           # rerun
  for a, b in [(0, 1), (1, 64), (63, 129), (700, 956), (3400, 3500), (n - 5, n)]:
    if b <= n:
      assert torch.equal(gpu.fd_distances(x[a:b].contiguous(), seeds, 255.0), full[a:b]), (a, b)
  rolled = torch.cat([x[n // 2:], x[:n // 2]])                                          # other offsets, other mates
  assert torch.equal(gpu.fd_distances(rolled, seeds, 255.0), torch.cat([full[n // 2:], full[:n // 2]]))
  assert torch.equal(gpu.fd_distances(x, seeds[:37].contiguous(), 255.0), full[:, :37])
  torch.cuda.synchronize()


@pytest.mark.gpu
def test_range_and_counts(gpu):
  check_counts_and_range(gpu)
  rs = np.random.RandomState(2)
  x = _images(rs, 3000, 3072)
  dist = gpu.fd_distances(_dev(gpu, x), _dev(gpu, x[:100]), 255.0)
  host = dist.cpu().numpy().ravel()
  lo, hi = gpu.fd_range(dist)
  assert lo == np.min(host[np.nonzero(host)]) and hi == np.max(host)
  edges = lo * ((hi / lo) ** np.linspace(0, 1, 1000))[1:]
  edges[500] = host[1234]                                     # a distance exactly on an edge
  edges = np.sort(edges)
  assert np.array_equal(gpu.fd_counts(dist, edges), oracle.counts(host, edges))


@pytest.mark.gpu
@pytest.mark.parametrize("dim,want,tol", REFERENCE_CASES)
def test_reference_cases(gpu, dim, want, tol):
  got, expect = check_reference_cases(gpu, dim, want, tol)
  assert abs(got - expect) <= 1e-9, (got, expect)


@pytest.mark.gpu
def test_end_to_end_at_cifar_size(gpu):
  rs = np.random.RandomState(9)
  z = rs.uniform(size=(10000, 5))
  x = (1 / (1 + np.exp(-(z @ rs.randn(5, 3072))))).astype(np.float32)         # a 5-dimensional manifold in [0, 1]
  x255 = np.float32(255.0) * x
  got = _fd().compute_fractal_dimension(x255, random_state=3)
  want = oracle.fractal_dimension(x255, np.random.RandomState(3).randint(10000, size=100))
  assert abs(got - want) <= 1e-9 * max(1.0, abs(want)), (got, want)
  from compare_gan_b200.tape import DT
  assert _fd().compute_fractal_dimension(DT(_dev(gpu, x255.reshape(10000, 32, 32, 3))), random_state=3) == got


@pytest.mark.gpu
def test_argument_errors(gpu):
  import torch
  lib = gpu.lib()
  x = torch.zeros(10, 4, device="cuda")
  out = torch.zeros(10, 3, dtype=torch.float64, device="cuda")
  cnt = torch.zeros(5, dtype=torch.int64, device="cuda")
  X, O, C = x.data_ptr(), out.data_ptr(), cnt.data_ptr()
  cases = {
      "cgan_fd_distances": ([dict(out=None), dict(x=None), dict(seeds=None), dict(n=0), dict(s=0), dict(d=0),
                             dict(d=-1), dict(scale=float("nan")), dict(scale=float("inf"))],
                            lambda a: (a["out"], a["x"], a["n"], a["seeds"], a["s"], a["d"], a["scale"])),
      "cgan_fd_range": ([dict(out=None), dict(dist=None), dict(count=0), dict(count=-3)],
                        lambda a: (a["out"], a["dist"], a["count"])),
      "cgan_fd_counts": ([dict(cnt=None), dict(dist=None), dict(edges=None), dict(count=0), dict(nedges=0),
                          dict(nedges=8193)],
                         lambda a: (a["cnt"], a["dist"], a["count"], a["edges"], a["nedges"])),
  }
  for name, (bad, args) in cases.items():
    fn = lib.fn[name]
    for case in bad:
      a = dict(out=O, x=X, seeds=X, dist=O, edges=O, cnt=C, n=10, s=3, d=4, scale=1.0, count=30, nedges=5)
      a.update(case)
      assert fn(lib.ctx, *args(a)) == 1, (name, case)
      assert lib.fn["cgan_last_error"](lib.ctx).decode().startswith(name + ":"), (name, case)
  d = gpu.fd_distances(x, x[:3].contiguous())                 # the context is still usable
  assert gpu.fd_range(d)[1] == 0 and np.array_equal(gpu.fd_counts(d, [0.0, 1.0]), [0, 30])
  torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("conditional", [False, True])
def test_evaluation(gpu, conditional):
  check_evaluation(gpu, use_graph=True, conditional=conditional)
