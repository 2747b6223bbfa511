"""BigGAN-128 (`biggan_imagenet128`, math_mode 1, CUDA-graph replay) with and without recomputed blocks.

  python profiles/prof_biggan_batch256.py [--cycles N] [--rounds R]

Prints the card's name and power limit, then
  * at 64 images per GPU: the stash path and forced segments (every residual / non-local block of G and D recomputed in
    the backward pass, tape.segment), built side by side and timed alternately for R rounds of N cycles each: peak device
    memory (torch.cuda.max_memory_allocated above what was resident before the engine was built) and ms per cycle;
  * at 256 images per GPU (the reference's 2048 over 8 GPUs): which networks ModularGAN.build chose to segment, the peak
    memory and ms per cycle; then the same with forced segments.
A cycle is disc_iters = 2 D-updates and one G-update.  The numbers are quoted in DESIGN.md §6."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def build(batch, force):
  import torch
  from compare_gan_b200 import configs, datasets, gin_lite as gin, runner_lib
  from compare_gan_b200.gans import modular_gan
  gin.clear_config()
  gin.parse_config(configs.CONFIGS["biggan_imagenet128"])
  gin.parse_config("ModularGAN.math_mode = 1")
  options = runner_lib.get_options_dict()
  ds = datasets.get_dataset()
  saved = modular_gan.memory_budget
  if force:
    modular_gan.memory_budget = lambda: -1          # nothing fits: segment both networks
  torch.cuda.synchronize()
  base = torch.cuda.memory_allocated()
  torch.cuda.reset_peak_memory_stats()
  try:
    eng = options["gan_class"](dataset=ds, parameters=options, model_dir="/tmp/cgan_prof_biggan256").build(batch)
  finally:
    modular_gan.memory_budget = saved
  pred = getattr(eng, "predicted_stash", {})
  print("%d/GPU%s: recompute %s; predicted stash GB %s" % (batch, " (forced)" if force else "", eng.recompute, {
      "%s%s" % (k[0][0].upper(), "/seg" if k[1] else "") if isinstance(k, tuple) else k: round(v / 1e9, 2)
      for k, v in pred.items()}))
  sys.stdout.flush()
  rng = np.random.RandomState(0)
  inputs = [runner_lib.sample_cycle_inputs(eng, ds, batch, rng) for _ in range(2)]
  eng.set_inputs(*inputs[0])
  eng.capture(warmup=2)
  eng.run_cycle()
  torch.cuda.synchronize()
  peak = torch.cuda.max_memory_allocated() - base
  return {"eng": eng, "inputs": inputs, "peak_gb": peak / 1e9, "ms": []}


def time_cycles(r, n):
  import torch
  eng = r["eng"]
  st = torch.cuda.current_stream()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  eng.run_cycle()
  torch.cuda.synchronize()
  e0.record(st)
  for i in range(n):
    eng.set_inputs(*r["inputs"][i % 2])
    eng.run_cycle()
  e1.record(st)
  torch.cuda.synchronize()
  r["ms"].append(e0.elapsed_time(e1) / n)
  d, g = eng.read_losses()
  assert np.isfinite(d).all() and np.isfinite(g), (d, g)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--cycles", type=int, default=5)
  ap.add_argument("--rounds", type=int, default=3)
  args = ap.parse_args()
  import gc
  import torch
  from compare_gan_b200 import kernels as K
  K.init(0)
  card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                        capture_output=True, text=True).stdout.strip()
  total = torch.cuda.get_device_properties(0).total_memory
  print("card: %s (%.1f GB)" % (card, total / 1e9))
  out = {"card": card, "device_gb": total / 1e9}

  runs = {"stash": build(64, False), "segments": build(64, True)}
  assert runs["stash"]["eng"].recompute == {"generator": False, "discriminator": False}
  for _ in range(args.rounds):
    for name in ("stash", "segments"):
      time_cycles(runs[name], args.cycles)
  out["batch64"] = {}
  for name, r in runs.items():
    out["batch64"][name] = {"recompute": r["eng"].recompute, "peak_gb": r["peak_gb"], "ms_per_cycle": r["ms"]}
    print("64/GPU  %-9s recompute %-50s peak %6.2f GB  ms/cycle %s" % (name, r["eng"].recompute, r["peak_gb"],
                                                                      " ".join("%.1f" % m for m in r["ms"])))
  runs.clear()
  gc.collect()
  torch.cuda.empty_cache()

  out["batch256"] = {}
  for name, force in (("auto", False), ("segments", True)):     # one at a time: both do not fit side by side
    r = build(256, force)
    for _ in range(args.rounds):
      time_cycles(r, args.cycles)
    out["batch256"][name] = {"recompute": r["eng"].recompute, "peak_gb": r["peak_gb"], "ms_per_cycle": r["ms"]}
    print("256/GPU %-9s recompute %-50s peak %6.2f GB  ms/cycle %s" % (name, r["eng"].recompute, r["peak_gb"],
                                                                      " ".join("%.1f" % m for m in r["ms"])))
    del r
    gc.collect()
    torch.cuda.empty_cache()
  print(json.dumps(out))


if __name__ == "__main__":
  main()
