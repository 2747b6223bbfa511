"""What the resnet_stl (48x48) and resnet30 (128x128) architectures cost at the reference's width (ch 64).

* the CUDA-graph-replayed training cycle of each (batch 64, disc_iters 5, math_mode 1, non-saturating loss, spectral
  norm in D, batch norm in G), timed with CUDA events;
* every filter-gradient shape of the resnet_stl cycle (kernels.CONV_TRACE), timed alone with CUDA events in math_mode 1
  (the path it takes there) and in math_mode 0 (the exact-fp32 gather-GEMM, the yard-stick), with its FLOPs and, on the
  wgmma kernel, its MMA row use (real pixel rows over the rows of the k-blocks, from the box rule of csrc/wgrad_tc.cu);
* resnet30's share of device time in the exact-fp32 SIMT contractions (gather_gemm_kernel) and the streaming image-side
  kernels (thin.cu), from torch.profiler over one eager cycle.

Writes OUT_DIR/prof_resnet_stl_resnet30.json with the card's name and power limit.

  python profiles/prof_resnet_stl_resnet30.py [--cycles 3] [--iters 20] [--out OUT_DIR]
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

BATCH = 64
ARCHS = {"resnet_stl": ("resnet_stl_arch", (48, 48, 3)), "resnet30": ("resnet30_arch", (128, 128, 3))}


def build(arch, image_shape):
  from compare_gan_b200 import datasets, gin_lite as gin
  from compare_gan_b200.gans import modular_gan
  gin.clear_config()
  gin.parse_config("G.batch_norm_fn = @batch_norm\nD.spectral_norm = True\nloss.fn = @non_saturating\n"
                   "penalty.fn = @no_penalty\nModularGAN.math_mode = 1")
  ds = datasets.ImageDatasetV2("synthetic", image_shape[0], image_shape[2], None, 100)
  params = {"architecture": arch, "z_dim": 128, "lambda": 1, "disc_iters": 5, "seed": 0}
  eng = modular_gan.ModularGAN(dataset=ds, parameters=params, model_dir="/tmp/cgan_prof_resnet_stl_resnet30")
  eng.build(BATCH)
  rs = np.random.RandomState(1)
  imgs = [rs.rand(BATCH, *image_shape).astype(np.float32) for _ in range(6)]
  zs = [rs.uniform(-1, 1, (BATCH, 128)).astype(np.float32) for _ in range(6)]
  eng.set_inputs(imgs, zs)
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


def box(n, h, w):
  """The k-block box of csrc/wgrad_tc.cu for an n x h x w grid: box32, else the fewest-k-block box of <= 32 pixels."""
  b = min(w, 32)
  if 32 % b == 0 and w % b == 0:
    hh = min(32 // b, h)
    ni = 32 // (b * hh)
    if h % hh == 0 and b * hh * ni == 32 and n % ni == 0:
      return b, hh, ni
  best = None
  for b in range(min(w, 32), 0, -1):
    for hh in range(min(32 // b, h), 0, -1):
      ni = min(32 // (b * hh), n)
      kb = -(-w // b) * -(-h // hh) * -(-n // ni)
      if best is None or kb < best[0]:
        best = (kb, b, hh, ni)
  return best[1:]


def wgrad_grid(n, h, w, stride, up):
  """The pixel grid the filter-gradient kernel sums over: dY's grid, or one sub-pixel phase of it."""
  oh, ow = (2 * h, 2 * w) if up else (-(-h // stride), -(-w // stride))
  return (n, oh // 2, ow // 2) if up else (n, oh, ow)


def time_wgrad(key, math_mode, iters):
  _, n, h, w, cin, cout, kh, kw, stride, up = key
  d = K.conv_desc(n, h, w, cin, cout, kh, kw, stride, bool(up))
  rs = np.random.RandomState(0)
  oh, ow = (2 * h, 2 * w) if up else (-(-h // stride), -(-w // stride))
  x = K.from_numpy(rs.standard_normal((n, h, w, cin)).astype(np.float32))
  dy = K.from_numpy(rs.standard_normal((n, oh, ow, cout)).astype(np.float32))
  dw = K.empty(kh, kw, cin, cout)
  K.set_math_mode(math_mode)
  call = lambda: K._call("conv2d_wgrad_ex", ctypes.byref(d), x.ptr, dy.ptr, 0, dw.ptr)
  call()
  path = _lib.PATH_NAMES[K.lib().get_option(_lib.OPT_LAST_PATH)]
  ms = events_ms(call, iters)
  K.set_math_mode(1)
  return ms, path


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--cycles", type=int, default=3)
  ap.add_argument("--iters", type=int, default=20)
  ap.add_argument("--out", default="prof_resnet_stl_resnet30_out")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("prof_resnet_stl_resnet30.py needs a CUDA device")
  K.init(0)
  card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                        text=True).stdout.strip().splitlines()[0]
  print(card)
  result = {"card": card, "batch": BATCH, "disc_iters": 5, "math_mode": 1, "ch": 64, "cycle_ms": {}}
  from torch.profiler import ProfilerActivity, profile
  for name, (arch, shape) in ARCHS.items():
    eng = build(arch, shape)
    K.CONV_TRACE = {}
    eng.run_cycle()
    trace = dict(K.CONV_TRACE)
    K.CONV_TRACE = None
    if name == "resnet30":
      eng.run_cycle()
      with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.run_cycle()
        torch.cuda.synchronize()
      total = simt = thin = 0.0
      for e in prof.key_averages():
        t = e.device_time_total
        total += t
        if "gather_gemm" in e.key:
          simt += t
        elif "_thin" in e.key and "thin_tc" not in e.key:
          thin += t
      result["resnet30_eager_cycle_device_us"] = total
      result["resnet30_share_simt_fp32"] = simt / total
      result["resnet30_share_thin_fp32"] = thin / total
      result["resnet30_paths"] = {"%s" % (k,): v[0] for k, v in sorted(trace.items())}
      print("resnet30 eager cycle: %.1f ms of kernels, %.1f %% gather-GEMM (simt_fp32), %.1f %% thin fp32"
            % (total / 1e3, 100 * simt / total, 100 * thin / total))
    eng.capture(warmup=2)
    times = [events_ms(eng.run_cycle, 1) for _ in range(args.cycles)]
    result["cycle_ms"][name] = {"median": float(np.median(times)), "all": times}
    print("%-10s cycle %.2f ms (median of %d graph-replayed cycles)" % (name, float(np.median(times)), args.cycles))
    if name == "resnet_stl":
      rows = []
      for key, rec in sorted(trace.items()):
        if key[0] != "wgrad":
          continue
        _, n, h, w, cin, cout, kh, kw, stride = key
        # CONV_TRACE keys an up-sampling convolution by its virtual (up-sampled) input; in resnet_stl those are exactly
        # the generator's (batch BATCH) convolutions that halve the width
        up = int(n == BATCH and cin == 2 * cout)
        if up:
          h, w = h // 2, w // 2
        k = ("wgrad", n, h, w, cin, cout, kh, kw, stride, up)
        oh, ow = (2 * h, 2 * w) if up else (-(-h // stride), -(-w // stride))
        flops = 2.0 * n * oh * ow * cin * cout * kh * kw / (4 if up else 1)     # taps over zero-inserted pixels excluded
        ms1, path1 = time_wgrad(k, 1, args.iters)
        ms0, path0 = time_wgrad(k, 0, args.iters)
        row = {"shape": list(k), "path": path1, "ms": ms1, "tflop_per_s": flops / ms1 / 1e9, "gather_gemm_ms": ms0,
               "gather_gemm_path": path0, "speedup": ms0 / ms1}
        if path1 == "tcgen05_tf32" and cin >= 64:
          gn, gh, gw = wgrad_grid(n, h, w, stride, up)
          bw, bh, bni = box(gn, gh, gw)
          kblocks = -(-gw // bw) * -(-gh // bh) * -(-gn // bni)
          row["box"], row["mma_row_use"] = [bw, bh, bni], gn * gh * gw / (32.0 * kblocks)
        rows.append(row)
        print("%-55s %-13s %8.3f ms %6.1f TFLOP/s  math_mode 0: %8.3f ms (%s)  rows %s"
              % (k, path1, ms1, row["tflop_per_s"], ms0, path0, row.get("mma_row_use")))
      result["resnet_stl_wgrad"] = rows
    del eng
    torch.cuda.empty_cache()
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "prof_resnet_stl_resnet30.json"), "w") as f:
    json.dump(result, f, indent=1)


if __name__ == "__main__":
  main()
