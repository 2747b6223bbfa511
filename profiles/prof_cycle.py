"""Where the time of the flagship cycle goes, kernel by kernel: the `resnet_cifar10` workload at batch 256, math_mode 1,
built as bench.py builds it, run eagerly (no CUDA graph, so every kernel shows up on its own) under torch.profiler with
CUDA activities.  Prints the device time per kernel name with its share of the summed kernel time and its launch count,
and writes the same table as JSON to OUT_DIR/prof_cycle.json.

The shares are what this is for.  Profiling and eager launches slow the host side, so the step time comes from bench.py,
not from here.

  python profiles/prof_cycle.py [--cycles 3] [--warmup 2] [--out OUT_DIR]
"""
import argparse
import collections
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

from bench import build_engine
from compare_gan_b200 import kernels as K, runner_lib


def short_name(name):
  """Kernel name without `void`, anonymous namespaces and the parameter list; template arguments stay (conv_tc_kernel<256,
  1> and conv_tc_kernel<128, 2> are different launches).  Copies and fills (`Memcpy HtoD (Pinned -> Device)`) keep
  their names."""
  if name.startswith(("Memcpy", "Memset")):
    return name
  name = re.sub(r"\(anonymous namespace\)::", "", name)
  if name.startswith("void "):
    name = name[5:]
  depth = 0
  for i, ch in enumerate(name):
    if ch == "<":
      depth += 1
    elif ch == ">":
      depth -= 1
    elif ch == "(" and depth == 0 and i > 0:
      return name[:i]
  return name


def table(events, cycles):
  per = collections.defaultdict(lambda: [0.0, 0])
  for e in events:
    if e.device_type != torch.autograd.DeviceType.CUDA:
      continue
    row = per[short_name(e.name)]
    row[0] += e.time_range.elapsed_us()
    row[1] += 1
  total = sum(r[0] for r in per.values())
  rows = [{"kernel": k, "ms_per_cycle": us / 1e3 / cycles, "share": us / total, "launches_per_cycle": n / cycles}
          for k, (us, n) in sorted(per.items(), key=lambda kv: -kv[1][0])]
  return rows, total / 1e3 / cycles


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--cycles", type=int, default=3)
  ap.add_argument("--warmup", type=int, default=2)
  ap.add_argument("--out", default="prof_cycle_out")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("prof_cycle.py needs a CUDA device")
  K.init(0)
  eng, ds, _ = build_engine("resnet_cifar10", 256, seed=0, math_mode=1)
  eng.set_inputs(*runner_lib.sample_cycle_inputs(eng, ds, 256, np.random.RandomState(1000)))
  for _ in range(args.warmup):
    eng.run_cycle()
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(args.cycles):
      eng.run_cycle()
    torch.cuda.synchronize()
  rows, total_ms = table(prof.events(), args.cycles)
  props = torch.cuda.get_device_properties(0)
  print("%s, %d SMs; %d eager cycles; summed kernel time %.2f ms per cycle" % (props.name, props.multi_processor_count,
                                                                               args.cycles, total_ms))
  print("%-72s %10s %7s %9s" % ("kernel", "ms/cycle", "share", "launches"))
  for r in rows:
    print("%-72s %10.3f %6.1f%% %9.0f" % (r["kernel"][:72], r["ms_per_cycle"], 100 * r["share"], r["launches_per_cycle"]))
  os.makedirs(args.out, exist_ok=True)
  with open(os.path.join(args.out, "prof_cycle.json"), "w") as f:
    json.dump({"device": props.name, "cycles": args.cycles, "kernel_ms_per_cycle": total_ms, "kernels": rows}, f, indent=1)


if __name__ == "__main__":
  main()
