"""Device time of the generator condition number (GeneratorConditionNumberTask) at the evaluation batch of 64 samples.
Reports the card, its power limit and maximum SM clock (read in the same run), then per generator:
  - the tangent pass: G in exact fp32 (math_mode 0) on every z column of all 64 samples, in chunks of
    jacobian_conditioning.TANGENT_ROWS tangent images (host clock around work that ends in a synchronise, after a
    warm-up pass), and the peak device memory it allocated;
  - the Gram kernel (cgan_metric_tensor_f64) on the [64, z_dim, D] tangent output: CUDA events over repeated calls, its
    FLOPs 2 B k^2 D counted from the shapes, and that rate's share of the 67 TFLOP/s FP64 tensor-core data-sheet figure;
  - the whole task call (compute_generator_condition_number).

  python profiles/prof_jacobian.py [--nets resnet_cifar biggan128] [--out prof_jacobian_out/prof_jacobian.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

FP64_TC_DATASHEET = 67e12
B = 64

# (architecture, image shape, z_dim, gin bindings, conditional classes)
NETS = {
    "resnet_cifar": ("resnet_cifar_arch", (32, 32, 3), 128, ["G.batch_norm_fn = @batch_norm"], 0),
    "biggan128": ("resnet_biggan_arch", (128, 128, 3), 120,
                  ["G.batch_norm_fn = @conditional_batch_norm", "G.spectral_norm = True",
                   "spectral_norm.singular_value = 'auto'", "weights.initializer = 'orthogonal'"], 1000),
}


def card():
  try:
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                  text=True).strip().splitlines()[0]
    name, power, clock = [v.strip() for v in out.split(",")]
    return name, power, clock
  except (OSError, subprocess.CalledProcessError, ValueError, IndexError) as e:
    return "unknown (%s)" % e, "unknown", "unknown"


def build(name):
  from compare_gan_b200 import datasets
  from compare_gan_b200 import gin_lite as gin
  from compare_gan_b200.gans import modular_gan
  arch, shape, z_dim, bindings, classes = NETS[name]
  gin.clear_config()
  gin.parse_config("\n".join(bindings))
  ds = datasets.ImageDatasetV2("synthetic", shape[0], shape[2], classes or None, 100)
  gan = modular_gan.ModularGAN(dataset=ds, parameters={"architecture": arch, "z_dim": z_dim, "lambda": 1, "disc_iters": 1,
                                                       "seed": 0},
                               model_dir="/tmp/prof_jacobian", conditional=bool(classes))
  gan.build(B)
  return gan


def measure(name, reps):
  import torch
  from compare_gan_b200 import kernels as K
  from compare_gan_b200.metrics import jacobian_conditioning as jc
  gan = build(name)
  z, labels = jc._draw_latents(gan, B, np.random.RandomState(0))
  with jc._GeneratorPass(gan) as run:
    run(z[:2], None if labels is None else labels[:2])             # warm-up: modules, workspace
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.time()
    _, tangents = run(z, labels)
    torch.cuda.synchronize()
    pass_s = time.time() - t0
    peak = torch.cuda.max_memory_allocated() - base
  k, d = tangents.shape[1], tangents.shape[2]
  tangents = tangents.contiguous()
  K.metric_tensor_f64(tangents)
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(reps):
    K.metric_tensor_f64(tangents)
  b.record()
  b.synchronize()
  gram_ms = a.elapsed_time(b) / reps
  flops = 2.0 * B * k * k * d
  del tangents
  torch.cuda.synchronize()
  t0 = time.time()
  lc = jc.compute_generator_condition_number(gan, B, np.random.RandomState(0))
  torch.cuda.synchronize()
  task_s = time.time() - t0
  return {"net": name, "samples": B, "z_dim": k, "D": d, "tangent_rows_per_chunk": jc.TANGENT_ROWS,
          "tangent_pass_s": round(pass_s, 3), "tangent_pass_peak_alloc_gb": round(peak / 2 ** 30, 2),
          "gram_ms": round(gram_ms, 3), "gram_flops": flops, "gram_fp64_tflops": round(flops / (gram_ms * 1e-3) / 1e12, 2),
          "gram_share_of_67_datasheet": round(flops / (gram_ms * 1e-3) / FP64_TC_DATASHEET, 3),
          "task_s": round(task_s, 3), "log_condition_number_mean": float(np.mean(lc))}


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--nets", nargs="+", default=sorted(NETS))
  p.add_argument("--reps", type=int, default=20)
  p.add_argument("--out", default=os.path.join("prof_jacobian_out", "prof_jacobian.json"))
  args = p.parse_args()
  from compare_gan_b200 import kernels as K
  K.init(0)
  name, power, clock = card()
  res = {"card": name, "power_limit": power, "max_sm_clock": clock, "runs": [measure(n, args.reps) for n in args.nets]}
  print(json.dumps(res, indent=1))
  os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
  with open(args.out, "w") as f:
    json.dump(res, f, indent=1)


if __name__ == "__main__":
  main()
