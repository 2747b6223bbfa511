"""What the discriminator penalties cost on the `resnet_lsun-bedroom128` workload (resnet5 at 128x128, batch 64,
disc_iters 5, math_mode 1), built as bench.py builds it with `penalty.fn` rebound.

* the CUDA-graph-captured training cycle under no_penalty, wgangp_penalty, dragan_penalty and l2_penalty, timed with CUDA
  events in the same process, alternating between the four engines;
* DRAGAN's perturbation of the 64x128x128x3 real batch: the whole entry (the batch moments, then the elementwise pass)
  and the elementwise pass alone (12.6 MB read, 12.6 MB written), timed with CUDA events;
* the L2 forward and backward over the discriminator kernels of `biggan_imagenet128` (BigGAN-128 at full width), with
  the bytes they must move: the forward reads every kernel once, the backward reads the kernels and the gradient slots
  and writes the slots.

Bandwidths are against the H100 SXM data sheet's 3.35 TB/s.  Writes OUT_DIR/prof_penalties.json with the card's name
and power limit.

  python profiles/prof_penalties.py [--steps 5] [--rounds 3] [--iters 50] [--out OUT_DIR]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from compare_gan_b200 import kernels as K, runner_lib

WORKLOAD, BATCH = "resnet_lsun-bedroom128", 64
PENALTIES = ("no_penalty", "wgangp_penalty", "dragan_penalty", "l2_penalty")
HBM_BYTES_PER_S = 3.35e12


def build(workload, penalty, batch, cycle=True):
  """bench.build_engine with `penalty.fn` rebound (lambda stays the workload's 10)."""
  from compare_gan_b200 import configs, datasets, gin_lite as gin
  from compare_gan_b200.gans import modular_gan  # noqa: F401
  gin.clear_config()
  gin.parse_config(configs.CONFIGS[workload])
  gin.parse_config("ModularGAN.math_mode = 1\npenalty.fn = @%s" % penalty)
  options = runner_lib.get_options_dict()
  options["seed"] = 0
  ds = datasets.get_dataset()
  eng = options["gan_class"](dataset=ds, parameters=options, model_dir="/tmp/cgan_prof_penalties")
  eng.build(batch)
  if cycle:
    eng.set_inputs(*runner_lib.sample_cycle_inputs(eng, ds, batch, np.random.RandomState(1000)))
    eng.run_cycle()
    eng.capture(warmup=2)
  return eng


def events_ms(fn, n):
  st = torch.cuda.current_stream()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  e0.record(st)
  for _ in range(n):
    fn()
  e1.record(st)
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / n


def row(name, ms, nbytes, extra=None):
  r = {"kernel": name, "ms": ms, "bytes_needed": nbytes, "tb_per_s": nbytes / ms / 1e9,
       "share_of_3_35_tb_per_s": nbytes / ms / 1e9 / (HBM_BYTES_PER_S / 1e12)}
  r.update(extra or {})
  print("%-28s %9.4f ms  %7.1f MB  %6.2f TB/s  %5.1f %%" % (name, ms, nbytes / 1e6, r["tb_per_s"],
                                                        100 * r["share_of_3_35_tb_per_s"]))
  return r


def perturb_rows(iters):
  shape = (BATCH, 128, 128, 3)
  n = int(np.prod(shape))
  x = K.from_numpy(np.random.RandomState(0).rand(*shape).astype(np.float32))
  y, std, step = K.empty(*shape), K.empty(1), torch.zeros(1, dtype=torch.int32, device="cuda")
  entry = lambda: K._call("dragan_perturb", y.ptr, x.ptr, n, 7, step.data_ptr(), std.ptr)
  moments = K.empty(2)
  # the layer-norm moments of one sample spanning the batch: what the entry's first launch reads
  reduce = lambda: K._call("layer_norm_moments", moments.ptr, x.ptr, 1, n, 0.0)
  for _ in range(3):
    entry()
    reduce()
  t_entry, t_reduce = events_ms(entry, iters), events_ms(reduce, iters)
  return [row("dragan_perturb (2 launches)", t_entry, 3 * 4 * n),
          row("  batch moments", t_reduce, 4 * n),
          row("  elementwise pass", t_entry - t_reduce, 2 * 4 * n, {"derived": "entry minus the moments launch"})]


def l2_rows(iters):
  eng = build("biggan_imagenet128", "l2_penalty", 2, cycle=False)
  segs, flat = eng.d_kernels, eng.flat_d
  params = sum(flat["views"][k][1] for k in segs.kernels)
  out, scale = K.empty(1), K.from_numpy(np.array([0.1], np.float32))
  fwd = lambda: K._call("l2_penalty", out.ptr, flat["param"].ptr, segs.table.data_ptr(), segs.n)
  bwd = lambda: K._call("l2_penalty_bwd", flat["grad"].ptr, flat["param"].ptr, segs.table.data_ptr(), segs.n, scale.ptr,
                        1.0 / segs.n)
  for _ in range(3):
    fwd()
    bwd()
  info = {"kernels": segs.n, "kernel_params": params, "d_params": flat["total"]}
  print("BigGAN-128 D: %d kernels, %.1f M kernel parameters" % (segs.n, params / 1e6))
  return [row("l2_penalty", events_ms(fwd, iters), 4 * params, info),
          row("l2_penalty_bwd", events_ms(bwd, iters), 3 * 4 * params, info)]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--iters", type=int, default=50)
  ap.add_argument("--out", default="prof_penalties_out")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("prof_penalties.py needs a CUDA device")
  K.init(0)
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip().splitlines()[0]
  print(card)
  engines = {p: build(WORKLOAD, p, BATCH) for p in PENALTIES}
  times = {p: [] for p in engines}
  for _ in range(args.rounds):
    for p, eng in engines.items():
      times[p].append(events_ms(eng.run_cycle, args.steps))
  for p, v in times.items():
    print("%-15s cycle %.2f ms (median of %d rounds of %d graph-replayed cycles; all: %s)"
          % (p, float(np.median(v)), args.rounds, args.steps, ", ".join("%.2f" % t for t in v)))
  del engines
  torch.cuda.empty_cache()
  kernels = perturb_rows(args.iters) + l2_rows(args.iters)
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "prof_penalties.json"), "w") as f:
    json.dump({"card": card, "workload": WORKLOAD, "batch": BATCH, "math_mode": 1,
               "cycle_ms": {p: {"median": float(np.median(v)), "all": v} for p, v in times.items()},
               "kernels": kernels}, f, indent=1)


if __name__ == "__main__":
  main()
