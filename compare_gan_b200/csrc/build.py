"""Build libcgan_b200.so in-tree with nvcc for sm_90a (no torch headers, plain C-ABI)."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "libcgan_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=default", "-Wno-deprecated-gpu-targets"]


def sources():
  return sorted(glob.glob(os.path.join(HERE, "*.cu")))


def stale():
  if not os.path.exists(OUT):
    return True
  t = os.path.getmtime(OUT)
  deps = sources() + glob.glob(os.path.join(HERE, "*.cuh")) + [os.path.join(HERE, "..", "..", "include", "cgan_b200.h")]
  return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
  if not force and not stale():
    return OUT
  objs = []
  procs = []
  os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
  for src in sources():
    obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
    objs.append(obj)
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
    procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
  for cmd, p in procs:
    out, _ = p.communicate()
    if verbose or p.returncode != 0:
      sys.stderr.write(out.decode())
    if p.returncode != 0:
      raise RuntimeError("nvcc failed: " + " ".join(cmd))
  cmd = [NVCC, "-shared", "-o", OUT] + objs
  subprocess.check_call(cmd)
  return OUT


if __name__ == "__main__":
  print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
