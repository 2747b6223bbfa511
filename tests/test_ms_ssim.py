"""MS-SSIM (reference metrics/image_similarity.py, metrics/ms_ssim_score.py): the float64 restatement against the
reference's golden and an independent write-out, the task's batch selection, the device terms (cgan_ssim_terms)
against float64, their exactness properties, and the metric inside the evaluation loop."""
import json
import os

import numpy as np
import pytest
import scipy.ndimage

from tests import ms_ssim_oracle as oracle
from tests.abi_emulator import EmulatedLib, emulated_library, f32, i32

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "ms_ssim_golden.json")))["ms_ssim"]


def _images(rng, n, h, w, c=3):
  """Images whose pairs score spread over (0, 1): two smooth base images plus noise of several strengths."""
  yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
  bases = [127.5 + 100 * np.sin(6 * xx + 4 * yy)[..., None] * np.ones(c),
           127.5 + 90 * np.cos(9 * yy * xx + 2)[..., None] * np.linspace(0.6, 1.0, c)]
  out = []
  for i in range(n):
    noise = rng.randn(h, w, c) * (5, 20, 45, 80)[i % 4]
    out.append(np.clip(bases[(i // 4) % 2] + noise, 0, 255))
  return np.stack(out).astype(np.float32)


# ---- an independent float64 write-out: MATLAB fspecial window, scipy correlation, explicit pooling and pair loops ----

def _fspecial(size, sigma):
  ax = np.arange(size) - (size - 1) / 2.0
  g = np.exp(-(ax[:, None] ** 2 + ax[None, :] ** 2) / (2.0 * sigma ** 2))
  return g / g.sum()


def _valid_filter(plane, win):
  f = win.shape[0]
  full = scipy.ndimage.correlate(plane, win, mode="constant")
  o = f // 2
  return full[o:o + plane.shape[0] - f + 1, o:o + plane.shape[1] - f + 1]


def _pool(img):
  h, w, c = img.shape
  ho, wo = (h + 1) // 2, (w + 1) // 2
  out = np.zeros((ho, wo, c))
  for i in range(ho):
    for j in range(wo):
      rows, cols = [2 * i, min(2 * i + 1, h - 1)], [2 * j, min(2 * j + 1, w - 1)]
      out[i, j] = sum(img[r, q] for r in rows for q in cols) / 4.0
  return out


def _written_out_msssim(x, y, weights=oracle.WEIGHTS, size=11, sigma=1.5, max_val=255.0):
  c1, c2 = (0.01 * max_val) ** 2, (0.03 * max_val) ** 2
  x, y = x.astype(np.float64), y.astype(np.float64)
  per_channel = np.ones(x.shape[-1])
  for k, wgt in enumerate(weights):
    if k:
      x, y = _pool(x), _pool(y)
    win = _fspecial(min(size, x.shape[0], x.shape[1]), sigma)
    for ch in range(x.shape[-1]):
      a, b = x[..., ch], y[..., ch]
      ma, mb = _valid_filter(a, win), _valid_filter(b, win)
      va = _valid_filter(a * a, win) - ma * ma
      vb = _valid_filter(b * b, win) - mb * mb
      cov = _valid_filter(a * b, win) - ma * mb
      cs = (2 * cov + c2) / (va + vb + c2)
      lum = (2 * ma * mb + c1) / (ma * ma + mb * mb + c1)
      term = (lum * cs).mean() if k == len(weights) - 1 else cs.mean()
      per_channel[ch] *= max(term, 0.0) ** wgt
  return per_channel.mean()


def test_oracle_reproduces_the_reference_golden():
  imgs = np.stack([np.ones((64, 64, 3)), np.ones((64, 64, 3)) * 0.7, np.zeros((64, 64, 3))])
  got = oracle.compute_msssim(imgs, GOLDEN["num_batches"])
  assert abs(got - GOLDEN["expected"]) <= GOLDEN["tolerance"], got


@pytest.mark.parametrize("shape,unweighted", [((32, 32), False), ((64, 64), False), ((40, 36), False), ((32, 32), True)])
def test_oracle_matches_an_independent_write_out(shape, unweighted):
  imgs = _images(np.random.RandomState(0), 4, shape[0], shape[1])
  fn = oracle.multiscale_ssim_unweighted if unweighted else oracle.multiscale_ssim
  weights = [1] * 5 if unweighted else oracle.WEIGHTS
  for i, j in [(0, 1), (1, 2), (0, 3), (2, 3)]:
    want = _written_out_msssim(imgs[i], imgs[j], weights)
    got = fn(imgs[i], imgs[j])
    assert abs(got - want) <= 1e-12, (shape, i, j, got, want)
    assert 0.0 < want < 1.0


def test_oracle_exactness_symmetry_and_ordered_pair_formula():
  imgs = _images(np.random.RandomState(1), 4, 32, 32)
  assert oracle.multiscale_ssim(imgs[2], imgs[2]) == 1.0
  assert oracle.multiscale_ssim(imgs[0], imgs[3]) == oracle.multiscale_ssim(imgs[3], imgs[0])
  from compare_gan_b200.metrics import ms_ssim_score
  got = ms_ssim_score.compute_msssim(imgs, num_batches=1, batch_size=4, pair_scores=_oracle_pair_scores)
  assert abs(got - oracle.compute_msssim(imgs, 1)) <= 1e-12


def _oracle_pair_scores(batch, pairs):
  batch = np.asarray(batch, np.float64)
  return oracle.multiscale_ssim(batch[pairs[:, 0]], batch[pairs[:, 1]])


def test_task_batch_selection_and_errors():
  from compare_gan_b200.metrics import eval_task, ms_ssim_score
  seen = []

  def scores(batch, pairs):
    seen.append((int(batch[0, 0, 0, 0]), len(batch), len(pairs)))
    return np.full(len(pairs), float(batch[0, 0, 0, 0]))
  imgs = np.arange(23, dtype=np.float32)[:, None, None, None] * np.ones((1, 2, 2, 1), np.float32)
  assert ms_ssim_score.compute_msssim(imgs, num_batches=5, batch_size=4, pair_scores=scores) == np.mean([0, 4, 8, 12, 16])
  assert seen == [(0, 4, 6), (4, 4, 6), (8, 4, 6), (12, 4, 6), (16, 4, 6)]
  del seen[:]
  assert ms_ssim_score.compute_msssim(imgs[:11], num_batches=5, batch_size=4, pair_scores=scores) == 2.0   # whole batches
  assert seen == [(0, 4, 6), (4, 4, 6)]
  del seen[:]
  assert ms_ssim_score.compute_msssim(imgs[3:6], num_batches=5, batch_size=4, pair_scores=scores) == 3.0   # one short batch
  assert seen == [(3, 3, 3)]
  with pytest.raises(ValueError):
    ms_ssim_score.compute_msssim(imgs[:1], pair_scores=scores)
  task = ms_ssim_score.MultiscaleSSIMTask()
  assert task.images_needed == 320 and task._LABEL == "ms_ssim" and eval_task.EvalTask.images_needed == 0
  assert ms_ssim_score.MultiscaleSSIMTask(num_batches=2, batch_size=16).images_needed == 32


# ---- the device entry point, emulated on the CPU through the float64 oracle ----

def _emulated_ssim_terms(self, out, images, n, h, w, c, pairs, npairs, levels, filter_size, filter_width, max_val):
  x = f32(images, n * h * w * c).reshape(n, h, w, c)
  p = i32(pairs, 2 * npairs).reshape(npairs, 2)
  assert levels >= 1 and (min(h, w) >> (levels - 1)) >= 1 and p.min() >= 0 and p.max() < n
  t = oracle.terms(x[p[:, 0]], x[p[:, 1]], levels, filter_size, filter_width, max_val)
  f32(out, npairs * levels * c)[:] = t.astype(np.float32).ravel()


@pytest.fixture
def emulated(monkeypatch):
  monkeypatch.setattr(EmulatedLib, "cgan_ssim_terms", _emulated_ssim_terms, raising=False)
  from compare_gan_b200 import kernels as K
  with emulated_library():
    yield K


@pytest.fixture(scope="module")
def gpu():
  from compare_gan_b200 import kernels as K
  K.init(0)
  return K


def _all_pairs(n):
  return np.stack(np.triu_indices(n, 1), axis=1)


SHAPES = [(32, 32), (64, 64), (128, 128), (40, 36), (48, 80)]


def check_terms_against_float64(K, shape):
  h, w = shape
  imgs = _images(np.random.RandomState(h * 1000 + w), 8, h, w)
  pairs = _all_pairs(len(imgs))
  got = K.ssim_terms(K.from_numpy(imgs), pairs, 5, 11, 1.5, 255.0)
  want = oracle.terms(imgs[pairs[:, 0]], imgs[pairs[:, 1]])
  assert got.shape == want.shape == (len(pairs), 5, 3)
  err = np.abs(got - want).max()
  assert err <= 3e-4, (shape, err)
  # the final per-pair MS-SSIM: bounded by what a literal fp32 restatement loses on the same pairs
  from compare_gan_b200.metrics import image_similarity
  ms = image_similarity.combine(got, image_similarity._MSSSIM_WEIGHTS)
  ms64 = oracle.multiscale_ssim(imgs[pairs[:, 0]], imgs[pairs[:, 1]])
  t32 = oracle.terms(imgs[pairs[:, 0]], imgs[pairs[:, 1]], dtype=np.float32)
  loss32 = np.abs(image_similarity.combine(t32, image_similarity._MSSSIM_WEIGHTS) - ms64).max()
  assert np.abs(ms - ms64).max() <= max(2 * loss32, 1e-5), (shape, np.abs(ms - ms64).max(), loss32)
  assert ms64.min() < 0.5 and ms64.max() > 0.8, (ms64.min(), ms64.max())      # the cases cover the range


def check_bit_exactness(K):
  imgs = _images(np.random.RandomState(5), 6, 48, 40)
  x = K.from_numpy(imgs)
  pairs = _all_pairs(6)
  allp = K.ssim_terms(x, pairs, 5, 11, 1.5, 255.0)
  assert np.array_equal(allp, K.ssim_terms(x, pairs, 5, 11, 1.5, 255.0))                       # two runs
  k = 7
  assert np.array_equal(K.ssim_terms(x, pairs[k:k + 1], 5, 11, 1.5, 255.0)[0], allp[k])          # alone vs in the call
  assert np.array_equal(K.ssim_terms(x, pairs[::-1, ::-1], 5, 11, 1.5, 255.0)[::-1], allp)       # (j, i) == (i, j)
  same = K.ssim_terms(x, np.array([[i, i] for i in range(6)]), 5, 11, 1.5, 255.0)
  assert np.all(same == 1.0)
  from compare_gan_b200.metrics import image_similarity
  assert np.all(image_similarity.multiscale_ssim(imgs, imgs) == 1.0)


def check_multiscale_ssim_functions(K):
  imgs = _images(np.random.RandomState(6), 8, 64, 64)
  a, b = imgs[:4], imgs[4:]
  from compare_gan_b200.metrics import image_similarity
  for fn, ofn in [(image_similarity.multiscale_ssim, oracle.multiscale_ssim),
                  (image_similarity.multiscale_ssim_unweighted, oracle.multiscale_ssim_unweighted)]:
    got, want = fn(a, b), ofn(a, b)
    assert got.shape == (4,) and got.dtype == np.float64
    assert np.abs(got - want).max() <= 1e-4, (got, want)


@pytest.mark.parametrize("shape", SHAPES[:2] + SHAPES[3:4])
def test_terms_on_the_emulator(emulated, shape):
  check_terms_against_float64(emulated, shape)


def test_exactness_and_functions_on_the_emulator(emulated):
  check_bit_exactness(emulated)
  check_multiscale_ssim_functions(emulated)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
def test_terms_match_float64(gpu, shape):
  check_terms_against_float64(gpu, shape)


@pytest.mark.gpu
def test_terms_bit_exactness(gpu):
  check_bit_exactness(gpu)


@pytest.mark.gpu
def test_multiscale_ssim_functions(gpu):
  check_multiscale_ssim_functions(gpu)


@pytest.mark.gpu
def test_argument_errors(gpu):
  lib = gpu.lib()
  fn = lib.fn["cgan_ssim_terms"]
  x = gpu.from_numpy(np.zeros((3, 32, 32, 3), np.float32))
  out = gpu.empty(4, 5, 3)
  ok = np.array([[0, 1], [1, 2]], np.int32)
  bad = np.array([[0, 1], [1, 3]], np.int32)
  neg = np.array([[0, -1]], np.int32)
  cases = [
      dict(out=None), dict(images=None), dict(pairs=None), dict(n=0), dict(pairs=bad), dict(pairs=neg), dict(levels=0),
      dict(filter_size=0), dict(levels=7), dict(h=15, levels=5),
  ]
  for case in cases:
    a = dict(out=out.ptr, images=x.ptr, n=3, h=32, w=32, pairs=ok, levels=5, filter_size=11)
    a.update(case)
    pr = a["pairs"]
    npairs = 0 if pr is None else len(pr)
    rc = fn(lib.ctx, a["out"], a["images"], a["n"], a["h"], a["w"], 3, None if pr is None else pr.ctypes.data, max(npairs, 1),
            a["levels"], a["filter_size"], 1.5, 255.0)
    assert rc == 1, (case, rc)
    assert fn is lib.fn["cgan_ssim_terms"] and lib.fn["cgan_last_error"](lib.ctx).decode().startswith("cgan_ssim_terms:"), case
  gpu.ssim_terms(x, ok, 5, 11, 1.5, 255.0)        # the context is still usable
  import torch
  torch.cuda.synchronize()


def check_evaluation(K, use_graph):
  """evaluate() with MS-SSIM next to FID / IS: the score equals the oracle on the regenerated samples, the graph path
  equals the eager one, and FID / IS are bit-identical to a run without the MS-SSIM task."""
  from compare_gan_b200 import eval_gan_lib
  from compare_gan_b200.metrics import fid_score, inception_score, ms_ssim_score
  from tests.gpu_util import make_pair
  eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True)
  base = [fid_score.FIDScoreTask(), inception_score.InceptionScoreTask()]
  tasks = base + [ms_ssim_score.MultiscaleSSIMTask(batch_size=16, num_batches=2)]
  real = np.random.RandomState(5).rand(64, 32, 32, 3).astype(np.float32)
  kw = dict(num_averaging_runs=1, num_samples=144 if use_graph else 64, batch_size=32, seed=7, real_images=real)
  res = eval_gan_lib.evaluate(eng, tasks, use_graph=use_graph, **kw)
  for key in ("ms_ssim_mean", "ms_ssim_std", "ms_ssim_list"):
    assert key in res
  without = eval_gan_lib.evaluate(eng, base, use_graph=use_graph, **kw)
  for key in ("fid_score_mean", "inception_score_mean"):
    assert res[key] == without[key], key
  if use_graph:
    eager = eval_gan_lib.evaluate(eng, tasks, use_graph=False, **kw)
    assert res["ms_ssim_mean"] == eager["ms_ssim_mean"]
  rs = np.random.RandomState(7)
  imgs = eval_gan_lib.generate_batch(eng, 32, rs).cpu().astype(np.float64) * 255.0
  want = oracle.compute_msssim(imgs, 2)
  assert abs(res["ms_ssim_mean"] - want) <= 1e-4 * max(1.0, abs(want)), (res["ms_ssim_mean"], want)


@pytest.mark.gpu
def test_evaluation_with_ms_ssim(gpu):
  check_evaluation(gpu, use_graph=True)


def test_evaluation_with_ms_ssim_on_the_emulator(emulated):
  check_evaluation(emulated, use_graph=False)


# ---- sharded evaluation: the score of rank 0's images, broadcast ----

def _rank_worker(rank, world, port, q):
  import torch.distributed as dist
  os.environ["MASTER_ADDR"] = "127.0.0.1"
  os.environ["MASTER_PORT"] = str(port)
  dist.init_process_group("gloo", rank=rank, world_size=world)
  EmulatedLib.cgan_ssim_terms = _emulated_ssim_terms
  from compare_gan_b200 import eval_utils
  from compare_gan_b200.metrics import ms_ssim_score
  with emulated_library():
    from compare_gan_b200 import kernels as K
    imgs = _images(np.random.RandomState(10 + rank), 6, 32, 32)       # every rank holds different samples
    sample = eval_utils.EvalDataSample(K.from_numpy(imgs))
    got = ms_ssim_score.MultiscaleSSIMTask(num_batches=1, batch_size=6).run_after_session(sample, None)["ms_ssim"]
    local = ms_ssim_score.compute_msssim(imgs, 1, 6, pair_scores=_oracle_pair_scores)
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
  assert res[0][0] == res[1][0]
  assert abs(res[0][0] - res[0][1]) <= 1e-6 and res[0][1] != res[1][1]
