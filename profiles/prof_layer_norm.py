"""What layer norm costs in the discriminator of the `resnet_lsun-bedroom128` workload (resnet5 at 128x128, batch 64,
WGAN-GP with lambda 10, disc_iters 5, math_mode 1), built as bench.py builds it, plus `D.layer_norm = True`.

* the CUDA-graph-captured training cycle with and without layer norm, timed with CUDA events in the same process,
  alternating between the two engines;
* each layer-norm entry (moments, apply, backward, double backward) at every layer-norm shape of that discriminator,
  timed alone with CUDA events, with the bandwidth it achieves on the bytes the algorithm needs (each tensor it must
  read or write, once) against the H100 SXM data sheet's 3.35 TB/s.

Writes OUT_DIR/prof_layer_norm.json with the card's name and power limit.

  python profiles/prof_layer_norm.py [--steps 5] [--rounds 3] [--iters 50] [--out OUT_DIR]
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
HBM_BYTES_PER_S = 3.35e12
# (h, w, c) of ln1 / ln2 of the discriminator blocks B0..B5 at 128x128 (resnet5.py: ch 64, multipliers 1,2,4,4,8,8)
SHAPES = [(128, 128, 3), (128, 128, 64), (64, 64, 64), (64, 64, 128), (32, 32, 128), (32, 32, 256), (16, 16, 256),
          (16, 16, 256), (8, 8, 256), (8, 8, 512), (4, 4, 512), (4, 4, 512)]


def build(layer_norm):
  """bench.build_engine plus the D.layer_norm binding."""
  from compare_gan_b200 import configs, datasets, gin_lite as gin
  from compare_gan_b200.gans import modular_gan  # noqa: F401
  gin.clear_config()
  gin.parse_config(configs.CONFIGS[WORKLOAD])
  gin.parse_config("ModularGAN.math_mode = 1\nD.layer_norm = %s" % layer_norm)
  options = runner_lib.get_options_dict()
  options["seed"] = 0
  ds = datasets.get_dataset()
  eng = options["gan_class"](dataset=ds, parameters=options, model_dir="/tmp/cgan_prof_layer_norm")
  eng.build(BATCH)
  eng.set_inputs(*runner_lib.sample_cycle_inputs(eng, ds, BATCH, np.random.RandomState(1000)))
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


def kernel_table(iters):
  rows = []
  rng = np.random.RandomState(0)
  for h, w, c in SHAPES:
    if any(r["shape"] == [BATCH, h, w, c] for r in rows):
      continue
    n, span = BATCH, h * w * c
    x, g, wv = (K.from_numpy(rng.standard_normal((n, h, w, c)).astype(np.float32)) for _ in range(3))
    gamma, beta = K.from_numpy(np.ones(c, np.float32)), K.zeros(c)
    stats, y, dx, d_g, d_x = K.empty(2 * n), K.empty(n, h, w, c), K.empty(n, h, w, c), K.empty(n, h, w, c), K.empty(n, h, w, c)
    dgamma, dbeta, d_gamma = K.empty(c), K.empty(c), K.empty(c)
    act = 1 | (K._lib.ACT_ROUND_TF32 if c > 4 else 0)          # fused ReLU; TF32 store where a tensor-core conv consumes it
    nbytes = 4 * n * span
    entries = [
        ("moments", lambda: K._call("layer_norm_moments", stats.ptr, x.ptr, n, span, K.LN_EPS), nbytes),
        ("apply", lambda: K._call("layer_norm_apply", y.ptr, x.ptr, n, span, c, stats.ptr, gamma.ptr, beta.ptr, act),
         2 * nbytes),
        ("bwd", lambda: K._call("layer_norm_bwd", dx.ptr, dgamma.ptr, dbeta.ptr, g.ptr, x.ptr, n, span, c, stats.ptr,
                                gamma.ptr, 0), 3 * nbytes),
        ("bwd_bwd", lambda: K._call("layer_norm_bwd_bwd", d_g.ptr, d_x.ptr, d_gamma.ptr, wv.ptr, g.ptr, x.ptr, n, span, c,
                                    stats.ptr, gamma.ptr, 0), 5 * nbytes),
    ]
    for name, fn, need in entries:
      for _ in range(3):
        fn()
      ms = events_ms(fn, iters)
      rows.append({"entry": name, "shape": [n, h, w, c], "ms": ms, "bytes_needed": need,
                   "tb_per_s": need / ms / 1e9, "share_of_3_35_tb_per_s": need / ms / 1e9 / (HBM_BYTES_PER_S / 1e12)})
      print("%-8s %-20s %8.4f ms  %6.2f TB/s  %5.1f %%" % (name, (n, h, w, c), ms, rows[-1]["tb_per_s"],
                                                         100 * rows[-1]["share_of_3_35_tb_per_s"]))
  return rows


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--iters", type=int, default=50)
  ap.add_argument("--out", default="prof_layer_norm_out")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("prof_layer_norm.py needs a CUDA device")
  K.init(0)
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip().splitlines()[0]
  print(card)
  engines = {"without_ln": build(False), "with_ln": build(True)}
  times = {k: [] for k in engines}
  for _ in range(args.rounds):
    for k, eng in engines.items():
      times[k].append(events_ms(eng.run_cycle, args.steps))
  for k, v in times.items():
    print("%-10s cycle %.2f ms (median of %d rounds of %d graph-replayed cycles; all: %s)"
          % (k, float(np.median(v)), args.rounds, args.steps, ", ".join("%.2f" % t for t in v)))
  del engines
  torch.cuda.empty_cache()
  rows = kernel_table(args.iters)
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "prof_layer_norm.json"), "w") as f:
    json.dump({"card": card, "workload": WORKLOAD, "batch": BATCH, "math_mode": 1,
               "cycle_ms": {k: {"median": float(np.median(v)), "all": v} for k, v in times.items()},
               "kernels": rows}, f, indent=1)


if __name__ == "__main__":
  main()
