"""Launch geometry A/B for the tensor-core convolutions: times the forward, input-gradient and filter-gradient launches of
the resnet_cifar10 cycle (batch 256; the discriminator sees 512 images) and of BigGAN-128 (batch 64) under two builds
of the library, alternately, in one call.  Each build is a source tree with its own compiled libcgan_b200.so (for
instance the parent commit checked out next to this one); a child process per (round, tree) imports the package from
that tree, so the two builds never share a process.

Per shape and direction it reports the column tile, pixel tiles per CTA, halo kernel and CTAs per SM each launch
reported (the filter gradient, which reports no geometry, is timed at the default and at one work unit per CTA), whether the two builds' results are bit-identical, the median time over the rounds, the useful FLOPs and their share of the H100 SXM data-sheet dense TF32 rate (495 TFLOP/s).  CUDA
events on the launching stream, 3 warm-ups + 10 timed launches per entry.  The card name, power limit and SM clock are
read in the same call.

Epilogue axis: the forward and the input gradient are timed bare ("fwd": a zero bias, which stays in L1; "dgrad": no
epilogue) and with the epilogue operands the cycle gives them, read from HBM: "fwd+res" adds a bias and a residual of
the output's shape (the last convolution of a residual block; not for the up-sampling convolutions, which never take
one), "dgrad+mask" gates the result with a ReLU mask (leak 0) and stores it TF32-rounded (the fused ReLU backward).  The
"gap" column is the epilogue row's time minus its bare row's time.

  python profiles/tile_ab.py --tree PARENT_TREE --tree . [--rounds 3] [--out tile_ab_out]
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

TF32_PEAK_TFLOPS = 495.0

# (label, batch, h, cin, cout, k, upsample): every convolution of the resnet_cifar10 generator (256 channels), the
# discriminator's 128-channel ones, and the BigGAN-128 layers (3x3 and 1x1 shortcuts) whose 768 / 1536 columns take
# 256-wide column tiles
SHAPES = [
    ("cifar G up 3x3 256->256 4->8", 256, 4, 256, 256, 3, True),
    ("cifar G up 3x3 256->256 8->16", 256, 8, 256, 256, 3, True),
    ("cifar G up 3x3 256->256 16->32", 256, 16, 256, 256, 3, True),
    ("cifar G 3x3 256->256 @8", 256, 8, 256, 256, 3, False),
    ("cifar G 3x3 256->256 @16", 256, 16, 256, 256, 3, False),
    ("cifar G 3x3 256->256 @32", 256, 32, 256, 256, 3, False),
    ("cifar G up 1x1 256->256 4->8", 256, 4, 256, 256, 1, True),
    ("cifar G up 1x1 256->256 8->16", 256, 8, 256, 256, 1, True),
    ("cifar G up 1x1 256->256 16->32", 256, 16, 256, 256, 1, True),
    ("cifar D 3x3 128->128 @32", 512, 32, 128, 128, 3, False),
    ("cifar D 1x1 128->128 @32", 512, 32, 128, 128, 1, False),
    ("cifar D 3x3 128->128 @16", 512, 16, 128, 128, 3, False),
    ("cifar D 3x3 128->128 @8", 512, 8, 128, 128, 3, False),
    ("biggan G up 3x3 1536->1536 4->8", 64, 4, 1536, 1536, 3, True),
    ("biggan G 3x3 1536->1536 @8", 64, 8, 1536, 1536, 3, False),
    ("biggan G up 3x3 1536->768 8->16", 64, 8, 1536, 768, 3, True),
    ("biggan G 3x3 768->768 @16", 64, 16, 768, 768, 3, False),
    ("biggan D 3x3 384->768 @16", 128, 16, 384, 768, 3, False),
    ("biggan D 3x3 768->768 @16", 128, 16, 768, 768, 3, False),
    ("biggan D 3x3 768->1536 @8", 128, 8, 768, 1536, 3, False),
    ("biggan D 3x3 1536->1536 @4", 128, 4, 1536, 1536, 3, False),
    ("biggan G up 1x1 1536->1536 4->8", 64, 4, 1536, 1536, 1, True),
    ("biggan G up 1x1 1536->768 8->16", 64, 8, 1536, 768, 1, True),
    ("biggan D 1x1 384->768 @16", 128, 16, 384, 768, 1, False),
    ("biggan D 1x1 768->1536 @8", 128, 8, 768, 1536, 1, False),
]


def child(tree):
  sys.path.insert(0, os.path.abspath(tree))
  import numpy as np
  import torch
  from compare_gan_b200 import _lib, kernels as K, tape

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

  K.init(0)
  K.set_math_mode(1)
  lib = K.lib()
  ctas_key = getattr(_lib, "OPT_LAST_TC_CTAS_PER_SM", None)

  def digest(t):
    return hashlib.sha1(np.ascontiguousarray(t.cpu()).tobytes()).hexdigest()[:12]

  def geometry():
    g = "bn%d mt%d%s" % (lib.get_option(_lib.OPT_LAST_TC_BN), lib.get_option(_lib.OPT_LAST_TC_MT),
                         " halo" if lib.get_option(_lib.OPT_LAST_TC_HALO) else "")
    if ctas_key is not None:
      g += " %d/SM" % lib.get_option(ctas_key)
    return g

  rows = []
  for label, b, h, cin, cout, k, up in SHAPES:
    x, w, bias = rand(b, h, h, cin), rand(k, k, cin, cout), K.zeros(cout)
    d = K.conv_desc(b, h, h, cin, cout, k, k, 1, up, "SAME")
    dy = rand(b, d.oh, d.ow, cout)
    ep_bias = rand(cout)
    res = None if up else rand(b, d.oh, d.ow, cout)
    mask = (rand(b, h, h, cin), 0.0)
    taps = k * k / 4.0 if up else k * k        # useful taps per output pixel (the zeros of the upsampling are skipped)
    flop = 2.0 * b * d.oh * d.ow * taps * cin * cout
    with tape.no_record():
      for pre in (False, True):                 # operands rounded in the kernel / already TF32-rounded by their producer
        x.tf32 = dy.tf32 = K.tf32_on() if pre else False
        suffix = " pre" if pre else ""
        ops = [("fwd", lambda: K.conv2d(x, w, bias, upsample=up)), ("dgrad", lambda: K.conv2d_dgrad(d, dy, w))]
        if res is not None:
          ops.append(("fwd+res", lambda: K.conv2d(x, w, ep_bias, upsample=up, residual=res)))
        ops.append(("dgrad+mask", lambda: K.conv2d_dgrad(d, dy, w, round_out=True, relu_mask=mask)))
        for op, fn in ops:
          ms = timed(fn)
          rows.append({"shape": label, "op": op + suffix, "ms": ms, "gflop": flop / 1e9, "geometry": geometry(),
                       "digest": digest(fn())})
        for mt in (2, 1):
          lib.set_option(_lib.OPT_TC_MT, mt)
          fn = lambda: K.conv2d_wgrad(d, x, dy)
          ms = timed(fn)
          rows.append({"shape": label, "op": "wgrad%s" % suffix, "ms": ms, "gflop": flop / 1e9,
                       "geometry": "tc_mt %d" % mt, "digest": digest(fn())})
        lib.set_option(_lib.OPT_TC_MT, 2)
    del x, w, dy, res, mask
    torch.cuda.empty_cache()
  print(json.dumps({"device": torch.cuda.get_device_name(0), "rows": rows}))


def card():
  try:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError) as e:
    return "nvidia-smi unavailable (%s)" % e


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--tree", action="append", default=[], help="source tree with a built library (give two)")
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--out", default="tile_ab_out")
  ap.add_argument("--child", help=argparse.SUPPRESS)
  args = ap.parse_args()
  if args.child:
    return child(args.child)
  if len(args.tree) != 2:
    raise SystemExit("give two --tree arguments")
  info = {"card_before": card(), "trees": args.tree, "rounds": args.rounds}
  runs = {t: [] for t in args.tree}
  for r in range(args.rounds):
    for t in args.tree:
      out = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", t], capture_output=True, text=True)
      if out.returncode != 0:
        sys.stderr.write(out.stdout + out.stderr)
        raise SystemExit("child for %s failed" % t)
      runs[t].append(json.loads(out.stdout.strip().splitlines()[-1]))
  info["card_after"] = card()
  info["device"] = runs[args.tree[0]][0]["device"]
  table = []
  for i, row in enumerate(runs[args.tree[0]][0]["rows"]):
    entry = {"shape": row["shape"], "op": row["op"], "gflop": row["gflop"]}
    for j, t in enumerate(args.tree):
      ms = [run["rows"][i]["ms"] for run in runs[t]]
      key = "ab"[j]
      entry[key + "_geometry"] = runs[t][0]["rows"][i]["geometry"]
      entry[key + "_ms"] = statistics.median(ms)
      entry[key + "_spread"] = max(ms) - min(ms)
      entry[key + "_tf32_share"] = row["gflop"] / entry[key + "_ms"] / TF32_PEAK_TFLOPS      # GFLOP / ms = TFLOP/s
    entry["same_bits"] = len({run["rows"][i]["digest"] for t in args.tree for run in runs[t]}) == 1
    table.append(entry)
  bare = {(e["shape"], e["op"]): e for e in table}
  for e in table:
    if "+" in e["op"]:
      op, _, rest = e["op"].partition("+")
      pre = " pre" if rest.endswith(" pre") else ""
      b = bare[(e["shape"], op + pre)]
      for key in "ab":
        e[key + "_gap"] = e[key + "_ms"] - b[key + "_ms"]
  print("%s | %s -> %s" % (info["device"], info["card_before"], info["card_after"]))
  print("A = %s, B = %s, median of %d rounds" % (args.tree[0], args.tree[1], args.rounds))
  print("%-34s %-15s %8s | %-28s %8s %6s %7s | %-28s %8s %6s %7s | %6s %s" % (
      "shape", "op", "GFLOP", "A geometry", "A ms", "A pk%", "A gap", "B geometry", "B ms", "B pk%", "B gap", "B/A",
      "bits"))
  gap = lambda e, key: "%7.3f" % e[key + "_gap"] if key + "_gap" in e else "%7s" % "-"
  for e in table:
    print("%-34s %-15s %8.1f | %-28s %8.3f %5.1f%% %s | %-28s %8.3f %5.1f%% %s | %6.3f %s" % (
        e["shape"], e["op"], e["gflop"], e["a_geometry"], e["a_ms"], 100 * e["a_tf32_share"], gap(e, "a"),
        e["b_geometry"], e["b_ms"], 100 * e["b_tf32_share"], gap(e, "b"), e["b_ms"] / e["a_ms"],
        "same" if e["same_bits"] else "DIFFER"))
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "tile_ab.json"), "w") as f:
    json.dump({"info": info, "rows": table}, f, indent=1)


if __name__ == "__main__":
  main()
