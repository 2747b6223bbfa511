"""What self-modulated batch norm (`G.batch_norm_fn = @self_modulated_batch_norm`, num_hidden 32) costs.

* the CUDA-graph-captured training cycle with `@batch_norm` and with `@self_modulated_batch_norm` on `resnet_cifar10`
  (batch 64, disc_iters 5) and `sndcgan_celebahq128` (batch 64; its g_bn1 normalises 131,072 channels), timed with
  CUDA events in the same process, alternating between the engines;
* the modulation entries at sndcgan's g_bn1 (N 64, z 128, H 32, C 131,072) under torch.profiler, with the bytes and
  FLOPs each needs, computed from the shapes;
* an A/B against the same MLP composed of kernels.matmul / bias_add / relu (built here only), forward and backward,
  timed with CUDA events, so that the fused kernels' benefit is measured rather than assumed.

Writes OUT_DIR/prof_self_modulation.json with the card's name and power limit.

  python profiles/prof_self_modulation.py [--steps 5] [--rounds 3] [--iters 50] [--out OUT_DIR]
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

from compare_gan_b200 import kernels as K, runner_lib, tape

BATCH = 64
WORKLOADS = ("resnet_cifar10", "sndcgan_celebahq128")
N, Z, H, C = 64, 128, 32, 131072          # sndcgan_celebahq128's g_bn1: seed 16 x 16 x 512 channels
HBM_BYTES_PER_S = 3.35e12


def build(workload, norm):
  from compare_gan_b200 import configs, datasets, gin_lite as gin
  from compare_gan_b200.gans import modular_gan  # noqa: F401
  gin.clear_config()
  gin.parse_config(configs.CONFIGS[workload])
  gin.parse_config("ModularGAN.math_mode = 1\nG.batch_norm_fn = @%s" % norm)
  options = runner_lib.get_options_dict()
  options["seed"] = 0
  options["disc_iters"] = 5
  ds = datasets.get_dataset()
  eng = options["gan_class"](dataset=ds, parameters=options, model_dir="/tmp/cgan_prof_self_modulation")
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


def layer_operands():
  rs = np.random.RandomState(0)
  dev = lambda a, req=True: K.from_numpy(a.astype(np.float32), req)
  z = dev(rs.uniform(-1, 1, (N, Z)), False)
  wh, bh = dev(rs.standard_normal((Z, H)) * 0.02), dev(np.zeros(H))
  wg, bg = dev(rs.standard_normal((H, C)) * 0.02), dev(np.ones(C))
  wb, bb = dev(rs.standard_normal((H, C)) * 0.02), dev(np.zeros(C))
  return z, [wh, bh, wg, bg, wb, bb]


def fused(z, w):
  return K.self_modulation(z, *w)


def composed(z, w):
  """The same MLP from the generic ops: 7 launches forward."""
  wh, bh, wg, bg, wb, bb = w
  h = K.relu(K.bias_add(K.matmul(z, wh), bh))
  return K.concat_rows(K.bias_add(K.matmul(h, wg), bg), K.bias_add(K.matmul(h, wb), bb))


def fwd_bwd(fn, z, w, dgb):
  out = fn(z, w)
  tape.backward([(out, dgb)], w, K.add_grad)


def needs():
  """Bytes each pass must move (every operand read once, every result written once) and its FLOPs."""
  f = 4
  fwd_bytes = f * (N * Z + Z * H + H + 2 * (H * C + C) + N * H + 2 * N * C)
  fwd_flops = 2 * N * Z * H + 2 * 2 * N * H * C
  bwd_bytes = f * (2 * N * C + N * H + N * Z + 2 * H * C + Z * H + 2 * (H * C + C) + Z * H + H)
  bwd_flops = 2 * 2 * N * H * C + 2 * 2 * N * H * C + 2 * N * Z * H
  return {"fwd": (fwd_bytes, fwd_flops), "bwd": (bwd_bytes, bwd_flops)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=5)
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--iters", type=int, default=50)
  ap.add_argument("--out", default="prof_self_modulation_out")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("prof_self_modulation.py needs a CUDA device")
  K.init(0)
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip().splitlines()[0]
  print(card)
  result = {"card": card, "batch": BATCH, "disc_iters": 5, "math_mode": 1, "cycle_ms": {}}
  for workload in WORKLOADS:
    engines = {norm: build(workload, norm) for norm in ("batch_norm", "self_modulated_batch_norm")}
    times = {k: [] for k in engines}
    for _ in range(args.rounds):
      for k, eng in engines.items():
        times[k].append(events_ms(eng.run_cycle, args.steps))
    result["cycle_ms"][workload] = {k: {"median": float(np.median(v)), "all": v} for k, v in times.items()}
    for k, v in times.items():
      print("%-20s %-26s cycle %.2f ms (median of %d rounds of %d graph-replayed cycles)"
            % (workload, k, float(np.median(v)), args.rounds, args.steps))
    del engines
    torch.cuda.empty_cache()

  z, w = layer_operands()
  dgb = K.from_numpy(np.random.RandomState(1).standard_normal((2 * N, C)).astype(np.float32))
  ab = {}
  for name, fn in (("fused", fused), ("composed", composed)):
    for _ in range(3):
      fwd_bwd(fn, z, w, dgb)
    with tape.no_record():
      f_ms = events_ms(lambda: fn(z, w), args.iters)
    fb_ms = events_ms(lambda: fwd_bwd(fn, z, w, dgb), args.iters)
    n0 = K.lib().launch_count()
    fwd_bwd(fn, z, w, dgb)
    ab[name] = {"fwd_ms": f_ms, "fwd_bwd_ms": fb_ms, "launches_fwd_bwd": K.lib().launch_count() - n0}
    print("%-9s forward %.4f ms, forward + backward %.4f ms, %d launches" % (name, f_ms, fb_ms,
                                                                          ab[name]["launches_fwd_bwd"]))
  result["ab_sndcgan_g_bn1"] = ab

  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(args.iters):
      fwd_bwd(fused, z, w, dgb)
    torch.cuda.synchronize()
  kernels = {}
  for e in prof.key_averages():
    if "sm_fwd" in e.key or "sm_bwd" in e.key:
      kernels[e.key] = {"count": e.count, "us_avg": e.device_time_total / max(e.count, 1)}
  need = needs()
  fwd_us = sum(v["us_avg"] for k, v in kernels.items() if "sm_fwd" in k)
  bwd_us = sum(v["us_avg"] for k, v in kernels.items() if "sm_bwd" in k)
  rows = {}
  for name, us in (("fwd", fwd_us), ("bwd", bwd_us)):
    nbytes, flops = need[name]
    rows[name] = {"us": us, "bytes_needed": nbytes, "flops": flops, "tb_per_s": nbytes / us / 1e6 if us else None,
                  "tflop_per_s": flops / us / 1e6 if us else None}
    print("%s: %.2f us, %.1f MB -> %.2f TB/s, %.2f GFLOP -> %.1f TFLOP/s" % (
        name, us, nbytes / 1e6, rows[name]["tb_per_s"] or 0, flops / 1e9, rows[name]["tflop_per_s"] or 0))
  result["kernels"] = {"shape": {"n": N, "z": Z, "hidden": H, "c": C}, "profiler": kernels, "passes": rows}
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "prof_self_modulation.json"), "w") as f:
    json.dump(result, f, indent=1)


if __name__ == "__main__":
  main()
