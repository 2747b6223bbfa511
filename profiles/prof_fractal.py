"""Device time of the fractal dimension's seed distances (cgan_fd_distances, S = 100 seeds) and the task's overhead on
one evaluation.  Reports the card, its power limit and maximum SM clock (read in the same run), then:
  - fd_distances per batch of 256 rows (the evaluation's fused batch) and over a whole run of N rows in batches of 256,
    CUDA events after a warm-up, with the FP64 FLOPs 2 N S D counted from the shapes.  Shares are given of the FP64
    pipe bound at the maximum SM clock (132 SMs x 64 FP64 lanes per cycle; each (row, seed, pixel) is a subtraction
    and an FMA, two pipe issues for its 2 FLOPs, so the bound is 132 * 64 * clock FLOP/s) and of the 34 TFLOP/s FP64
    data-sheet figure, which counts an FMA as two FLOPs;
  - one evaluate() at CIFAR size with and without FractalDimensionTask (host clock around work ending in a synchronise);
  - with --cpu, the reference formulation (scipy cdist + np.less.outer) on the host at N = 10000, D = 3072, labelled as a
    CPU figure with its thread count.

  python profiles/prof_fractal.py [--runs 10000:3072 50000:49152] [--eval-samples 10000] [--cpu]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

FP64_DATASHEET = 34e12
S = 100
BATCH = 256


def card():
  try:
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                  text=True).strip().splitlines()[0]
    name, power, clock = [v.strip() for v in out.split(",")]
    return name, power, float(clock.split()[0]) * 1e6
  except (OSError, subprocess.CalledProcessError, ValueError, IndexError) as e:
    return "unknown (%s)" % e, "unknown", None


def time_ms(fn, reps):
  import torch
  fn()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(reps):
    fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b) / reps


def rates(flops, ms, clock):
  r = flops / (ms * 1e-3)
  pipe = 132 * 64 * clock if clock else None
  return {"fp64_tflops": round(r / 1e12, 2), "share_of_pipe_bound": round(r / pipe, 3) if pipe else "not measured",
          "share_of_34_datasheet": round(r / FP64_DATASHEET, 3)}


def distances(K, n, d):
  import torch
  g = torch.Generator(device="cuda").manual_seed(n + d)
  x = torch.rand(n, d, device="cuda", generator=g)
  seeds = x[:S].contiguous()
  batch = x[:BATCH].contiguous()
  per_batch = time_ms(lambda: K.fd_distances(batch, seeds, 255.0), 50)

  def whole_run():
    for r0 in range(0, n, BATCH):
      K.fd_distances(x[r0:r0 + BATCH], seeds, 255.0)
  run = time_ms(whole_run, 2)
  one_call = time_ms(lambda: K.fd_distances(x, seeds, 255.0), 2)
  del x
  torch.cuda.empty_cache()
  return per_batch, run, one_call


def evaluation(n):
  import torch
  from compare_gan_b200 import eval_gan_lib
  from compare_gan_b200.metrics import fid_score, fractal_dimension, inception_score
  from tests.gpu_util import make_pair
  eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 64, d_sn=True)
  real = np.random.RandomState(5).rand(n, 32, 32, 3).astype(np.float32)
  base = [fid_score.FIDScoreTask(), inception_score.InceptionScoreTask()]
  with_fd = base + [fractal_dimension.FractalDimensionTask()]
  kw = dict(num_averaging_runs=1, num_samples=n, batch_size=64, seed=7, real_images=real)
  eval_gan_lib.evaluate(eng, with_fd, **dict(kw, num_samples=1024, real_images=real[:1024]))    # warm-up
  out = {"without": [], "with": []}
  for _ in range(2):                 # alternate the two configurations
    for key, tasks in (("without", base), ("with", with_fd)):
      torch.cuda.synchronize()
      t0 = time.time()
      res = eval_gan_lib.evaluate(eng, tasks, **kw)
      torch.cuda.synchronize()
      out[key].append((round(time.time() - t0, 3), round(res["eval_samples_per_sec"], 1),
                       res.get("fractal_dimension_mean")))
  return out


def cpu_reference(n, d):
  import scipy.spatial
  rs = np.random.RandomState(0)
  x = (rs.rand(n, d) * 255.0).astype(np.float32)
  t0 = time.time()
  dist = scipy.spatial.distance.cdist(x, x[rs.randint(n, size=S)]).flatten()
  t1 = time.time()
  lo, hi = np.min(dist[np.nonzero(dist)]), np.max(dist)
  edges = lo * ((hi / lo) ** np.linspace(0, 1, 1000))
  np.sum(np.less.outer(dist, edges[1:]), axis=0)
  t2 = time.time()
  return {"cdist_s": round(t1 - t0, 2), "less_outer_s": round(t2 - t1, 2),
          "threads": "1 (scipy cdist and np.less.outer run single-threaded; host has %d cores)" % os.cpu_count()}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--runs", nargs="+", default=["10000:3072", "50000:49152"])
  ap.add_argument("--eval-samples", type=int, default=10000)
  ap.add_argument("--cpu", action="store_true")
  args = ap.parse_args()
  from compare_gan_b200 import kernels as K
  K.init(0)
  name, power, clock = card()
  print(json.dumps({"card": name, "power_limit": power, "max_sm_clock_hz": clock}))
  for spec in args.runs:
    n, d = (int(v) for v in spec.split(":"))
    per_batch, run, one_call = distances(K, n, d)
    print(json.dumps({"n": n, "d": d, "s": S,
                      "batch_256_ms": round(per_batch, 3), "batch_256": rates(2.0 * BATCH * S * d, per_batch, clock),
                      "run_in_batches_ms": round(run, 2), "run": rates(2.0 * n * S * d, run, clock),
                      "one_call_ms": round(one_call, 2), "one_call": rates(2.0 * n * S * d, one_call, clock)}))
  if args.eval_samples:
    print(json.dumps({"evaluate_cifar": args.eval_samples, "wall_s_samples_per_s_fd": evaluation(args.eval_samples)}))
  if args.cpu:
    print(json.dumps({"cpu_reference_n10000_d3072": cpu_reference(10000, 3072)}))


if __name__ == "__main__":
  main()
