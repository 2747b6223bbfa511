"""What the 28x28x1 networks (infogan and sndcgan on MNIST-sized images) cost, and what the contractions routed onto the
tensor cores for them cost against the exact-fp32 paths they took before.

* every newly routed call, timed alone with CUDA events at batch 64 and 256: in math_mode 1 (the tensor-core path it
  takes now) and the same shape in math_mode 0 (the exact-fp32 kernels, the yard-stick).  The shapes are those of the
  two cycles: sndcgan's 4x4 stride-2 layers between 7x7 and 4x4 (g_dc2 forward and d_conv6 backward are both the input
  gradient of a 7 -> 4 convolution; their filter gradients share its shape too), and infogan's image layer between
  28x28x1 and 14x14x64 (g_dc4 forward and d_conv1's input gradient);
* the CUDA-graph-replayed training cycle of infogan and sndcgan on 28x28x1 images (batch 64, disc_iters 1, math_mode 1,
  non-saturating loss, spectral norm in D), timed with CUDA events.

Writes OUT_DIR/prof_grayscale28.json with the card's name and power limit.

  python profiles/prof_grayscale28.py [--cycles 10] [--iters 50] [--out OUT_DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from compare_gan_b200 import _lib, kernels as K

# (name, op, h, w, cin, cout, k): a stride-2 SAME convolution from h x w x cin to ceil(h/2) x ceil(w/2) x cout
CALLS = [
    ("sndcgan g_dc2 / d_conv6 input gradient", "dgrad", 7, 7, 256, 512, 4),
    ("sndcgan d_conv6 / g_dc2 filter gradient", "wgrad", 7, 7, 256, 512, 4),
    ("infogan g_dc4 / d_conv1 input gradient", "dgrad", 28, 28, 1, 64, 4),
]
BATCHES = (64, 256)
CYCLE_BATCH = 64
NETS = {"infogan_mnist": ("infogan_arch", 64), "sndcgan_mnist": ("sndcgan_arch", 128)}


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


def time_call(op, n, h, w, cin, cout, k, math_mode, iters):
  d = K.conv_desc(n, h, w, cin, cout, k, k, 2, False)
  rs = np.random.RandomState(0)
  x = K.from_numpy(rs.standard_normal((n, h, w, cin)).astype(np.float32))
  dy = K.from_numpy(rs.standard_normal((n, d.oh, d.ow, cout)).astype(np.float32))
  wt = K.from_numpy(rs.standard_normal((k, k, cin, cout)).astype(np.float32))
  out = K.empty(k, k, cin, cout) if op == "wgrad" else K.empty(n, h, w, cin)
  ep = K._epilogue()
  if op == "wgrad":
    call = lambda: K._call("conv2d_wgrad_ex", ctypes.byref(d), x.ptr, dy.ptr, 0, out.ptr)
  else:
    call = lambda: K._call("conv2d_dgrad_ex", ctypes.byref(d), dy.ptr, wt.ptr, ctypes.byref(ep), out.ptr)
  K.set_math_mode(math_mode)
  try:
    call()
    path = _lib.PATH_NAMES[K.lib().get_option(_lib.OPT_LAST_PATH)]
    for _ in range(3):
      call()
    ms = events_ms(call, iters)
  finally:
    K.set_math_mode(0)
  flops = 2.0 * n * d.oh * d.ow * cin * cout * k * k
  return {"path": path, "ms": ms, "tflop_per_s": flops / ms / 1e9}


def build(arch, z_dim):
  from compare_gan_b200 import datasets, gin_lite as gin
  from compare_gan_b200.gans import modular_gan
  gin.clear_config()
  gin.parse_config("G.batch_norm_fn = @batch_norm\nD.spectral_norm = True\nloss.fn = @non_saturating\n"
                   "penalty.fn = @no_penalty\nModularGAN.math_mode = 1")
  ds = datasets.get_dataset("mnist")
  params = {"architecture": arch, "z_dim": z_dim, "lambda": 1, "disc_iters": 1, "seed": 0}
  eng = modular_gan.ModularGAN(dataset=ds, parameters=params, model_dir="/tmp/cgan_prof_grayscale28")
  eng.build(CYCLE_BATCH)
  rs = np.random.RandomState(1)
  imgs = [rs.rand(CYCLE_BATCH, 28, 28, 1).astype(np.float32) for _ in range(2)]
  zs = [rs.uniform(-1, 1, (CYCLE_BATCH, z_dim)).astype(np.float32) for _ in range(2)]
  eng.set_inputs(imgs, zs)
  return eng


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--cycles", type=int, default=10)
  ap.add_argument("--iters", type=int, default=50)
  ap.add_argument("--out", default="prof_grayscale28_out")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("prof_grayscale28.py needs a CUDA device")
  K.init(0)
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip().splitlines()[0]
  print(card)
  result = {"card": card, "calls": [], "cycle_batch": CYCLE_BATCH, "disc_iters": 1, "math_mode": 1, "cycle_ms": {}}
  for name, op, h, w, cin, cout, k in CALLS:
    for n in BATCHES:
      tc = time_call(op, n, h, w, cin, cout, k, 1, args.iters)
      exact = time_call(op, n, h, w, cin, cout, k, 0, args.iters)
      row = {"call": name, "op": op, "shape": [n, h, w, cin, cout, k, k, 2], "math_mode_1": tc, "math_mode_0": exact,
             "speedup": exact["ms"] / tc["ms"]}
      result["calls"].append(row)
      print("%-42s n %3d  %-13s %8.4f ms %6.2f TFLOP/s | math_mode 0 %-10s %8.4f ms  -> x%.2f"
            % (name, n, tc["path"], tc["ms"], tc["tflop_per_s"], exact["path"], exact["ms"], row["speedup"]))
  K.set_math_mode(1)
  for name, (arch, z_dim) in NETS.items():
    eng = build(arch, z_dim)
    eng.run_cycle()
    eng.capture(warmup=2)
    times = [events_ms(eng.run_cycle, 1) for _ in range(args.cycles)]
    result["cycle_ms"][name] = {"median": float(np.median(times)), "all": times}
    print("%-14s cycle %.3f ms (median of %d graph-replayed cycles, batch %d)" % (name, float(np.median(times)),
                                                                                 args.cycles, CYCLE_BATCH))
    del eng
    torch.cuda.empty_cache()
  K.set_math_mode(0)
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "prof_grayscale28.json"), "w") as f:
    json.dump(result, f, indent=1)


if __name__ == "__main__":
  main()
