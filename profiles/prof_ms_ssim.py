"""Device time of the MS-SSIM task (MultiscaleSSIMTask: 5 batches of 64 generated images, every unordered pair of each
batch, 5 scales) at 32^2, 64^2 and 128^2, with CUDA events after warm-up.  Reports ms per call, pairs/s and the achieved
FP32 rate against the H100 SXM data-sheet 67 TFLOP/s, with an operation count computed from the shapes below, plus the
card name and power limit read in the same run.  With --literal it also times the reference's formulation on the same
GPU (all 64^2 ordered pairs, five 2-D 11x11 depthwise filterings per scale) through torch's conv2d: a comparison
only, nothing on the product path uses it.

  python profiles/prof_ms_ssim.py [--literal] [--out /tmp/prof_ms_ssim.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

PEAK_FP32 = 67e12       # H100 SXM data sheet, dense FP32, at up to 700 W
LEVELS, FILTER, BATCHES, BATCH = 5, 11, 5, 64


def level_shapes(h, w):
  out = []
  for _ in range(LEVELS):
    f = min(FILTER, h, w)
    out.append((h, w, f, h - f + 1, w - f + 1))
    h, w = (h + 1) // 2, (w + 1) // 2
  return out


def separable_flops(h, w, c):
  """FP32 operations of the engine's algorithm per call (BATCHES batches): per image and level two separable
  filterings (x' and x'^2), per unordered pair and level the product x'y', one separable filtering and the per-pixel
  luminance / cs evaluation (~12 operations).  A separable filtering of an h x w plane with an f-tap window costs
  h*ow*f + oh*ow*f FMAs = 2 FLOPs each."""
  pairs = BATCH * (BATCH - 1) // 2
  per_image = per_pair = 0
  for h_, w_, f, oh, ow in level_shapes(h, w):
    filt = 2 * (h_ * ow * f + oh * ow * f)
    per_image += c * (2 * filt + h_ * w_)
    per_pair += c * (filt + h_ * w_ + 12 * oh * ow)
  return BATCHES * (BATCH * per_image + pairs * per_pair)


def literal_fmas(h, w, c):
  """FMAs of the reference's formulation: B^2 ordered pairs, five full 2-D f x f filterings per pair and scale."""
  total = 0
  for _, _, f, oh, ow in level_shapes(h, w):
    total += 5 * c * oh * ow * f * f
  return BATCHES * BATCH * BATCH * total


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                     capture_output=True, text=True)
  return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "nvidia-smi unavailable: " + q.stderr.strip()


def seeded_images(n, h, w, c, seed):
  """Smooth base images plus noise of several strengths, in [0, 255] (pairs spread over (0, 1))."""
  rng = np.random.RandomState(seed)
  yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
  base = 127.5 + 100 * np.sin(6 * xx + 4 * yy)[..., None] * np.ones(c)
  noise = rng.randn(n, h, w, c) * rng.choice([5, 20, 45, 80], size=(n, 1, 1, 1))
  return np.clip(base + noise, 0, 255).astype(np.float32)


def time_events(fn, reps):
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(reps):
    fn()
  stop.record()
  stop.synchronize()
  return start.elapsed_time(stop) / reps


def literal_terms(x):
  """The reference's formulation on one batch [B,c,h,w] (fp32, no TF32): all B^2 ordered pairs, 2-D windows."""
  import torch.nn.functional as F
  b, c = x.shape[0], x.shape[1]
  p1, p2 = x.repeat(b, 1, 1, 1), x.repeat_interleave(b, dim=0)
  out = []
  for lvl in range(LEVELS):
    if lvl:
      pad = (0, p1.shape[3] % 2, 0, p1.shape[2] % 2)
      p1, p2 = [F.avg_pool2d(F.pad(t, pad, mode="replicate"), 2) for t in (p1, p2)]
    f = min(FILTER, p1.shape[2], p1.shape[3])
    g = torch.arange(f, dtype=torch.float32, device=x.device) - (f - 1) / 2.0
    g = -0.5 * g * g / 1.5 ** 2
    win = torch.softmax((g[None, :] + g[:, None]).reshape(-1), 0).reshape(1, 1, f, f).repeat(c, 1, 1, 1)
    red = lambda t: F.conv2d(t, win, groups=c)
    m0, m1 = red(p1), red(p2)
    num0, den0 = m0 * m1 * 2, m0 * m0 + m1 * m1
    cs = (red(p1 * p2) * 2 - num0 + 58.5225) / (red(p1 * p1 + p2 * p2) - den0 + 58.5225)
    out.append(((num0 + 6.5025) / (den0 + 6.5025) * cs if lvl == LEVELS - 1 else cs).mean(dim=(2, 3)))
  return torch.stack(out, 1)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--sizes", default="32,64,128")
  ap.add_argument("--reps", type=int, default=20)
  ap.add_argument("--literal", action="store_true")
  ap.add_argument("--out", default="")
  args = ap.parse_args()
  assert torch.cuda.is_available(), "prof_ms_ssim measures the H100: no CUDA device found"
  torch.backends.cudnn.allow_tf32 = False
  torch.backends.cuda.matmul.allow_tf32 = False
  from compare_gan_b200 import kernels as K
  from compare_gan_b200.metrics import ms_ssim_score
  K.init(0)
  dev_card = card()
  rows = []
  for s in [int(v) for v in args.sizes.split(",")]:
    imgs = K.from_numpy(seeded_images(BATCHES * BATCH, s, s, 3, seed=s))
    task_call = lambda: ms_ssim_score.compute_msssim(imgs, BATCHES, BATCH)
    score = task_call()
    task_call()                                                   # warm-up: workspace, module load
    ms = time_events(task_call, args.reps)
    flops = separable_flops(s, s, 3)
    pairs = BATCHES * BATCH * (BATCH - 1) // 2
    row = {"size": s, "ms_per_call": round(ms, 4), "pairs_per_s": round(pairs / (ms * 1e-3)), "score": score,
           "fp32_flop": flops, "achieved_tflops": round(flops / (ms * 1e-3) / 1e12, 3),
           "share_of_fp32_peak": round(flops / (ms * 1e-3) / PEAK_FP32, 4),
           "bound": "compute (fp32 FMA; the per-image maps stay in L2)",
           "literal_fma": literal_fmas(s, s, 3), "card": dev_card}
    if args.literal:
      x = imgs.t[:BATCH].permute(0, 3, 1, 2).contiguous()
      lit = lambda: literal_terms(x)
      lit()
      torch.cuda.synchronize()
      row["literal_ms_per_batch"] = round(time_events(lit, 3), 3)
      row["literal_ms_per_call"] = round(row["literal_ms_per_batch"] * BATCHES, 3)
      del x
      torch.cuda.empty_cache()
    rows.append(row)
    print(json.dumps(row), flush=True)
  if args.out:
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    with open(args.out, "w") as f:
      json.dump(rows, f, indent=1)


if __name__ == "__main__":
  main()
