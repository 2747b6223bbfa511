"""Device time of the PRD task (PRDScoreTask: compute_prd_from_embedding with 20 clusters, 10 runs x 10 seedings) on
seeded mixture features of N points per side, d = 2048.  Reports the card and its power limit (read in the same run),
CUDA-event time per C-ABI entry after a warm-up, the FP64 FLOPs of the distance contractions counted from the shapes
and iteration counts with their share of the 67 TFLOP/s FP64 tensor-core data-sheet figure, and, with --cpu, the
reference formulation (sklearn MiniBatchKMeans) on the host cores, labelled as a CPU figure.

  python profiles/prof_prd.py [--n 10000 50000] [--cpu]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

FP64_TC_PEAK = 67e12


def features(n, d, seed):
  rs = np.random.RandomState(seed)
  centers = np.abs(rs.randn(40, d)) * 0.3
  ref = np.abs(centers[rs.randint(40, size=n)] + 0.2 * rs.randn(n, d)).astype(np.float32)
  ev = np.abs(centers[rs.randint(28, size=n)] + 0.2 * rs.randn(n, d)).astype(np.float32)
  return ev, ref


def card():
  try:
    return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                   text=True).strip()
  except (OSError, subprocess.CalledProcessError) as e:
    return "unknown (%s)" % e


def timed_entries(K, n, d):
  """Runs the PRD clustering once, timing each entry with CUDA events.  Returns (ms per entry, FLOPs per entry, result)."""
  import torch
  from compare_gan_b200.metrics import prd_score
  times, flops = {"seed": 0.0, "finish": 0.0, "lloyd_step": 0.0}, {"seed": 0.0, "finish": 0.0, "lloyd_step": 0.0}
  wrapped = {}
  m = 2 * n

  def wrap(name, count):
    fn = getattr(K, "kmeans_" + name)
    wrapped[name] = fn

    def run(*args):
      flops[name] += count(*args)       # before the call: the Lloyd step changes the running groups
      a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      a.record()
      out = fn(*args)
      b.record()
      b.synchronize()
      times[name] += a.elapsed_time(b)
      return out
    setattr(K, "kmeans_" + name, run)
  # distance contractions: 2 m d FLOPs per (point, centre) evaluated
  wrap("seed", lambda x, u: 2.0 * m * d * u.shape[0] * (u.shape[1] - 1))
  wrap("finish", lambda x, c, n_eval: 2.0 * m * d * c.shape[0] * c.shape[1])
  wrap("lloyd_step", lambda x, c, labels, state, tol: 2.0 * m * d * int((state.cpu().numpy()[:, 0] == 0).sum()) * c.shape[1])
  ev, ref = features(n, d, 0)
  try:
    _, iters = prd_score._cluster_runs(ev, ref, 20, 10, 0)
  finally:
    for name, fn in wrapped.items():
      setattr(K, "kmeans_" + name, fn)
  return times, flops, iters


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--n", type=int, nargs="+", default=[10000, 50000])
  ap.add_argument("--d", type=int, default=2048)
  ap.add_argument("--cpu", action="store_true")
  args = ap.parse_args()
  import torch
  from compare_gan_b200 import kernels as K
  from compare_gan_b200.metrics import prd_score
  K.init(0)
  print("card:", card())
  for n in args.n:
    ev, ref = features(n, args.d, 0)
    prd_score.PRDScoreTask().run_after_session(type("S", (), {"activations": ev})(), type("S", (), {"activations": ref})())
    torch.cuda.synchronize()
    t0 = time.time()
    task = prd_score.PRDScoreTask().run_after_session(type("S", (), {"activations": ev})(),
                                                      type("S", (), {"activations": ref})())
    torch.cuda.synchronize()
    wall = time.time() - t0
    times, flops, iters = timed_entries(K, n, args.d)
    row = {"n_per_side": n, "d": args.d, "task_wall_s": round(wall, 3), "task": task, "lloyd_iterations": iters.tolist()}
    for name in times:
      row[name + "_ms"] = round(times[name], 2)
      row[name + "_fp64_tflops"] = round(flops[name] / (times[name] * 1e-3) / 1e12, 2) if times[name] else None
      row[name + "_share_of_67"] = round(flops[name] / (times[name] * 1e-3) / FP64_TC_PEAK, 3) if times[name] else None
    if args.cpu:
      try:
        import sklearn.cluster
        x = np.vstack([ev, ref]).astype(np.float64)
        t0 = time.time()
        sklearn.cluster.MiniBatchKMeans(n_clusters=20, n_init=10, random_state=0).fit(x)
        row["cpu_reference_one_fit_s"] = round(time.time() - t0, 2)
        row["cpu_reference_call_s_estimate_x10"] = round(10 * (time.time() - t0), 1)
        row["cpu_threads"] = os.cpu_count()
      except ImportError:
        row["cpu_reference_one_fit_s"] = "not measured (sklearn not importable)"
    print(json.dumps(row))


if __name__ == "__main__":
  main()
