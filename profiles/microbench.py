"""Per-kernel timing table on one GPU (no profiler): the convolution shapes of the resnet_cifar10 B=256 cycle and a few
BigGAN-128 ones (forward / input gradient / filter gradient, tensor-core path) as TFLOP/s, and the memory-bound kernel
families (BN forward / backward, ReLU, add, pooling, column sums) as algorithmic GB/s against the measured HBM peak.  CUDA events on
the launching stream, 3 warm-ups + 10 timed launches per entry; every operand set is larger than the 50 MB L2 or is
re-streamed between launches by the other operands of the same entry.

  python profiles/microbench.py [--math fp32] > microbench.txt
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from compare_gan_b200 import kernels as K, tape


def timed(fn, iters=10, warmup=3):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  st = torch.cuda.current_stream()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record(st)
  for _ in range(iters):
    fn()
  e1.record(st)
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / iters


def rand(*shape):
  return K.from_numpy((np.random.RandomState(sum(shape)).standard_normal(shape) * 0.1).astype(np.float32))


# (label, batch, h, cin, cout, k, stride, upsample)
CONVS = [
    ("cifar G B1 up 3x3 256->256 4->8", 256, 4, 256, 256, 3, 1, True),
    ("cifar G B2 up 3x3 256->256 8->16", 256, 8, 256, 256, 3, 1, True),
    ("cifar G B3 up 3x3 256->256 16->32", 256, 16, 256, 256, 3, 1, True),
    ("cifar G 3x3 256->256 @32", 256, 32, 256, 256, 3, 1, False),
    ("cifar G 1x1 up shortcut 256->256 16->32", 256, 16, 256, 256, 1, 1, True),
    ("cifar G out 3x3 256->3 @32", 256, 32, 256, 3, 3, 1, False),
    ("cifar D in 3x3 3->128 @32 (B=512)", 512, 32, 3, 128, 3, 1, False),
    ("cifar D 3x3 128->128 @32 (B=512)", 512, 32, 128, 128, 3, 1, False),
    ("cifar D 3x3 128->128 @16 (B=512)", 512, 16, 128, 128, 3, 1, False),
    ("cifar D 3x3 128->128 @8 (B=512)", 512, 8, 128, 128, 3, 1, False),
    ("cifar D 1x1 128->128 @32 (B=512)", 512, 32, 128, 128, 1, 1, False),
    ("biggan G 3x3 192->96 up 64->128 (B=64)", 64, 64, 192, 96, 3, 1, True),
    ("biggan D 3x3 96->96 @128 (B=128)", 128, 128, 96, 96, 3, 1, False),
    ("biggan D 3x3 1536->1536 @4 (B=512)", 512, 4, 1536, 1536, 3, 1, False),
    ("sndcgan D 4x4 s2 64->128 128->64 (B=256)", 256, 128, 64, 128, 4, 2, False),
]


def bench_convs(rows):
  for label, b, h, cin, cout, k, stride, up in CONVS:
    x = rand(b, h, h, cin)
    w = rand(k, k, cin, cout)
    bias = K.zeros(cout)
    d = K.conv_desc(b, h, h, cin, cout, k, k, stride, up, "SAME")
    dy = rand(b, d.oh, d.ow, cout)
    taps = k * k / 4.0 if up else k * k          # useful taps per OUTPUT pixel (the zeros of unpool are skipped)
    flop = 2.0 * b * d.oh * d.ow * taps * cin * cout
    bytes_io = 4.0 * (b * h * h * cin + b * d.oh * d.ow * cout)
    with tape.no_record():
      t_f = timed(lambda: K.conv2d(x, w, bias, stride=stride, upsample=up))
      t_d = timed(lambda: K.conv2d_dgrad(d, dy, w))
      t_w = timed(lambda: K.conv2d_wgrad(d, x, dy))
      # the same launches with operands flagged as already TF32-rounded by their producers (no in-kernel rounding pass)
      x.tf32 = dy.tf32 = K.tf32_on()
      t_fp = timed(lambda: K.conv2d(x, w, bias, stride=stride, upsample=up))
      t_dp = timed(lambda: K.conv2d_dgrad(d, dy, w))
      t_wp = timed(lambda: K.conv2d_wgrad(d, x, dy))
    rows.append({"kernel": label, "fwd_ms": t_f, "dgrad_ms": t_d, "wgrad_ms": t_w, "gflop": flop / 1e9,
                 "fwd_tflops": flop / t_f / 1e9, "dgrad_tflops": flop / t_d / 1e9, "wgrad_tflops": flop / t_w / 1e9,
                 "fwd_pre_ms": t_fp, "dgrad_pre_ms": t_dp, "wgrad_pre_ms": t_wp,
                 "fwd_pre_tflops": flop / t_fp / 1e9, "dgrad_pre_tflops": flop / t_dp / 1e9, "wgrad_pre_tflops": flop / t_wp / 1e9,
                 "fwd_hbm_gbs": bytes_io / t_f / 1e6})
    del x, w, dy
    torch.cuda.empty_cache()


def bench_memory_bound(rows):
  b, h, c = 256, 32, 256
  x, g = rand(b, h, h, c), rand(b, h, h, c)
  nbytes = 4.0 * b * h * h * c
  gamma, beta = K.from_numpy(np.ones(c, np.float32)), K.zeros(c)

  def entry(label, fn, passes):
    with tape.no_record():
      t = timed(fn)
    rows.append({"kernel": label, "ms": t, "algorithmic_gbs": passes * nbytes / t / 1e6, "passes": passes})

  entry("bn_train+relu fwd [256,32,32,256] (2 reads + 1 write)", lambda: K.bn_train(x, gamma, beta, 1e-5, relu_after=True), 3)
  entry("relu fwd (1 read + 1 write)", lambda: K.relu(x), 2)
  entry("add (2 reads + 1 write)", lambda: K.add(x, g), 3)
  entry("avgpool2 fwd (1 read + 1/4 write)", lambda: K.avgpool2(x), 1.25)
  entry("colsum [262144,256] (1 read)", lambda: K.colsum(K.reshape(x, -1, c)), 1)
  # BN backward through the tape: dy -> (dx, dgamma, dbeta)
  xr = K.from_numpy(x.cpu(), req=True)
  gr, br = K.from_numpy(np.ones(c, np.float32), req=True), K.from_numpy(np.zeros(c, np.float32), req=True)

  def bn_fwd_bwd():
    y = K.bn_train(xr, gr, br, 1e-5, relu_after=True)
    tape.backward([(y, g)], [xr, gr, br], K.add_grad)
  t = timed(bn_fwd_bwd)
  rows.append({"kernel": "bn_train+relu fwd+bwd (3 + ~5 passes)", "ms": t, "algorithmic_gbs": 8 * nbytes / t / 1e6, "passes": 8})


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--math", default="tf32", choices=["tf32", "fp32"])
  args = ap.parse_args()
  K.init(0)
  K.set_math_mode(1 if args.math == "tf32" else 0)
  rows = []
  bench_convs(rows)
  bench_memory_bound(rows)
  for r in rows:
    if "fwd_ms" in r:
      print("%-46s %8.1f GF  fwd %7.3f ms %6.1f TF/s (pre-rounded %7.3f ms %6.1f) | dgrad %7.3f ms %6.1f TF/s (%7.3f ms %6.1f) | "
            "wgrad %7.3f ms %6.1f TF/s (%7.3f ms %6.1f)" % (
                r["kernel"], r["gflop"], r["fwd_ms"], r["fwd_tflops"], r["fwd_pre_ms"], r["fwd_pre_tflops"], r["dgrad_ms"],
                r["dgrad_tflops"], r["dgrad_pre_ms"], r["dgrad_pre_tflops"], r["wgrad_ms"], r["wgrad_tflops"], r["wgrad_pre_ms"],
                r["wgrad_pre_tflops"]))
    else:
      print("%-62s %7.3f ms  %7.0f GB/s algorithmic" % (r["kernel"], r["ms"], r["algorithmic_gbs"]))
  print(json.dumps(rows))


if __name__ == "__main__":
  main()
