"""The fused self-attention kernels of math_mode 1 (csrc/attn_tc.cu) and the softmax / rowdot kernels of the composed
path (csrc/pointwise.cu), element by element against float64.

Attention.  Q, K, V and dO are drawn on grids of TF32 values: Q and K as integers of |n| <= 511 (a few up to 640) times a
power of two, V and dO as integers of |n| <= 255 times a power of two.  Every product of S = Q K^T and dP = dO V^T is then
exact in fp32 and so is every partial sum, in any order, so the kernels see the float64 scores.  The float64 reference is
plain softmax attention and its three gradients on those operands (D = rowsum(dO O) from the float64 O).  The verdict
is per element:

    |y - y64| <= TAU A + gamma(L) A + 1e-30,    TAU = 2^-10 (two TF32 units: the kernels round P and dS to TF32)

    O[i,c]   A = sum_j P_ij |V_jc|            L = 2 lk + 8  (P V, the normaliser sum, ex2, reciprocal, product)
    dV[j,c]  A = sum_i P_ij |dO_ic|           L = lq + 8
    dQ[i,:]  A = sum_j W_ij |K_j|             L = lk + dv + 8
    dK[j,:]  A = sum_i W_ij |Q_i|             L = lq + dv + 8
    W_ij = P_ij (|dP_ij| + Dabs_i),  Dabs_i = sum_c |dO_ic| sum_j P_ij |V_jc|

Dabs covers the error D inherits from the forward's TF32 probabilities (through O).  lse_i = m_i + log l_i is held to
8 u (|m_i| + |log l_i|) + 8 u + gamma(lk): a few ulp for the rounding of m log2e, logf and the final sum, the ex2.approx
error (the PTX ISA bounds ex2.approx.f32 by 2 ulp over its full range, 4 u) and the fp32 sum l; u = 2^-24.

Score regimes: diffuse (scores of std ~1.2), wide (std ~25: far keys fall below 2^-126 and ex2.approx.ftz flushes them),
offset (every score near -100: the max subtraction, lse far from 0), tied (identical keys: every P is exactly 1 / lk and
every key ties for the row maximum) and routing.  Routing gives key j the +-1 binary code of j in its first ceil(log2 lk)
channels and query i 4 times the code of its designated key pi(i), so pi(i) leads every other key by at least 8 and
O_i ~ V_pi(i), dV_j ~ sum over pi(i) = j of dO_i: a misplaced key, row, tile or image moves an element by about its own
size, which random scores hide (two swapped keys of 1024 diffuse ones move an output by ~1/1024 of its scale).  pi
designates every position of every 64-key tile (every key when lq >= lk) and differs per image.

Every GPU case keeps its inputs and outputs (lse too) inside NaN-sentinel guard bands, asserts CGAN_OPT_LAST_PATH and the
kernel counts (forward 1; backward 3: rowdot, the dQ kernel, the dK/dV kernel), and runs twice with bit-identical results.
Operands 4 or 8 bytes off the kernels' float4 / float2 alignment are refused with CGAN_ERR_UNSUPPORTED, nothing launched
and nothing written.

Softmax and rowdot (cgan_softmax_fwd / _bwd: the warp kernels at 1024 and 256 aligned columns, the block kernel
otherwise; cgan_rowdot): per element against float64 with gamma(L) bounds, expf at 2 ulp (the library is built without
fast math) and the relative error u |x - m| that the rounded difference x - m carries into exp.

The CPU tests show the criterion accepting the kernels' arithmetic model (tests/abi_emulator.py, attention_tf32_model)
and rejecting local defects, check the case table, and run every table on the emulator.  The module prints the worst
err / (TAU A) per attention output and err / bound per softmax / rowdot kernel of the GPU run."""
import math
import time

import numpy as np
import pytest

from compare_gan_b200 import _lib
from tests.abi_emulator import attention_tf32_model, emulated_library
from tests.test_simt_exact_gpu import SENTINEL, Guarded, assert_path, check_bound, emulated, gamma, seed_of, verify

TAU = 2.0 ** -10
U = 2.0 ** -24
TINY = 1e-30
FLUSH = 126 / math.log2(math.e)          # s - m below -87.3: 2^(x log2 e) < 2^-126, flushed by ex2.approx.ftz
WORST = {}          # output -> (worst err / (TAU A) or err / bound, case)


@pytest.fixture(scope="module", autouse=True)
def _report(pytestconfig):
  t0 = time.time()
  WORST.clear()
  yield
  if not WORST:
    return
  lines = ["fused attention: worst err / (TAU A), TAU = 2^-10; softmax / rowdot: worst err / bound (%.1f s):" % (
      time.time() - t0)]
  lines += ["  %-14s %.3e  (%s)" % (k, WORST[k][0], WORST[k][1]) for k in sorted(WORST)]
  capman = pytestconfig.pluginmanager.getplugin("capturemanager")
  tr = pytestconfig.pluginmanager.getplugin("terminalreporter")
  if capman is None or tr is None:
    print("\n".join(lines))
    return
  with capman.global_and_fixture_disabled():
    tr.ensure_newline()
    for line in lines:
      tr.write_line(line)


def record(K, what, ratio, case):
  if not emulated(K) and ratio >= WORST.get(what, (-1.0, ""))[0]:
    WORST[what] = (ratio, case)


# ---------------------------------------------------------------------------------------------------- attention cases

def nv_pad(dv):
  return (dv + 31) // 32 * 32


class Case(object):
  def __init__(self, batch, lq, lk, dk, dv, regime):
    self.batch, self.lq, self.lk, self.dk, self.dv, self.regime = batch, lq, lk, dk, dv, regime

  @property
  def id(self):
    return "b%d-q%d-k%d-dk%d-dv%d-%s" % (self.batch, self.lq, self.lk, self.dk, self.dv, self.regime)

  def code_bits(self):
    return int(math.ceil(math.log2(self.lk)))


C = Case
CASES = [
    C(1, 128, 128, 4, 16, "diffuse"),       # one CTA per direction; NV 32 padded
    C(1, 128, 128, 4, 32, "wide"),
    C(3, 128, 128, 8, 48, "routing"),       # lq = lk = 128: a single dK/dV CTA per image
    C(3, 256, 512, 12, 64, "routing"),      # lq < lk
    C(2, 512, 256, 16, 80, "routing"),      # lq > lk; NV 96 padded
    C(2, 384, 640, 20, 96, "offset"),
    C(1, 256, 1024, 28, 112, "routing"),    # NV 128 padded
    C(2, 640, 384, 32, 128, "diffuse"),
    C(2, 4096, 1024, 24, 96, "diffuse"),    # BigGAN-128's non-local blocks
    C(2, 4096, 1024, 24, 96, "routing"),
    C(1, 4096, 1024, 12, 48, "wide"),
    C(1, 4096, 1024, 12, 48, "routing"),
    C(300, 128, 128, 8, 16, "routing"),     # a few hundred images of one CTA each
    C(2, 256, 256, 16, 64, "tied"),
    C(3, 128, 256, 32, 128, "wide"),
    C(1, 128, 512, 4, 112, "tied"),
    C(2, 256, 128, 4, 64, "offset"),
    C(2, 128, 384, 24, 32, "offset"),
]


def grid(rng, shape, sigma, step, top):
  """sigma N(0, 1) on the grid step * n, |n| <= top (TF32 values: |n| < 2^11)."""
  return (np.clip(np.rint(sigma * rng.standard_normal(shape) / step), -top, top) * step).astype(np.float32)


def designations(rng, lq, lk):
  """pi: the key each query routes to.  lq >= lk: every key, lq // lk or more times.  lq < lk: lq / (lk / 64) keys of
  every 64-key tile, at positions shifted by 7 per tile so that together they cover all 64; shuffled over the queries."""
  if lq >= lk:
    keys = np.arange(lq) % lk
  else:
    tiles = lk // 64
    r = np.arange(lq)
    t = r % tiles
    keys = t * 64 + (r // tiles + 7 * t) % 64
  return rng.permutation(keys)


def draw(c, salt=0):
  """(q, k, v, dout, pi) of the case; pi is None outside the routing regime."""
  rng = np.random.RandomState(seed_of(c.id, salt))
  b, lq, lk, dk, dv = c.batch, c.lq, c.lk, c.dk, c.dv
  step = 1.0 / 64
  diffuse = math.sqrt(1.2 / math.sqrt(dk))
  pi = None
  if c.regime == "diffuse":
    q, k = grid(rng, (b, lq, dk), diffuse, step, 511), grid(rng, (b, lk, dk), diffuse, step, 511)
  elif c.regime == "wide":
    sw = math.sqrt(25.0 / math.sqrt(dk))
    q, k = grid(rng, (b, lq, dk), sw, 1.0 / 16, 511), grid(rng, (b, lk, dk), sw, 1.0 / 16, 511)
  elif c.regime == "offset":
    rest = math.sqrt(1.2 / math.sqrt(max(dk - 1, 1)))
    q, k = grid(rng, (b, lq, dk), rest, step, 511), grid(rng, (b, lk, dk), rest, step, 511)
    q[:, :, 0], k[:, :, 0] = 10.0, -10.0
  elif c.regime == "tied":
    q = grid(rng, (b, lq, dk), diffuse, step, 511)
    k = np.repeat(grid(rng, (b, 1, dk), diffuse, step, 511), lk, axis=1)
  else:
    nb = c.code_bits()
    assert dk >= nb, "%s: %d channels cannot route %d keys" % (c.id, dk, lk)
    codes = 1.0 - 2.0 * ((np.arange(lk)[:, None] >> np.arange(nb)[None, :]) & 1)
    q, k = grid(rng, (b, lq, dk), 0.25, step, 511), grid(rng, (b, lk, dk), 0.25, step, 511)
    pi = np.stack([designations(rng, lq, lk) for _ in range(b)])
    k[:, :, :nb] = codes
    q[:, :, :nb] = 4.0 * codes[pi]
  v, dout = grid(rng, (b, lk, dv), 1.0, 1.0 / 32, 255), grid(rng, (b, lq, dv), 1.0, 1.0 / 32, 255)
  return q, k, v, dout, pi


def reference64(q, k, v, dout):
  """Softmax attention and its gradients in float64, per image, with A of every output and (m, log l) of every row."""
  out = {n: [] for n in ("out", "lse", "dq", "dk", "dv", "A_out", "A_dq", "A_dk", "A_dv", "m", "logl")}
  for qi, ki, vi, gi in zip(*(a.astype(np.float64) for a in (q, k, v, dout))):
    s = qi @ ki.T
    m = s.max(1, keepdims=True)
    e = np.exp(s - m)
    l = e.sum(1, keepdims=True)
    p = e / l
    o = p @ vi
    a_o = p @ np.abs(vi)
    dp = gi @ vi.T
    d = (gi * o).sum(1, keepdims=True)
    ds = p * (dp - d)
    w = p * (np.abs(dp) + (np.abs(gi) * a_o).sum(1, keepdims=True))
    for name, val in (("out", o), ("lse", (m + np.log(l))[:, 0]), ("dq", ds @ ki), ("dk", ds.T @ qi), ("dv", p.T @ gi),
                      ("A_out", a_o), ("A_dq", w @ np.abs(ki)), ("A_dk", w.T @ np.abs(qi)),
                      ("A_dv", p.T @ np.abs(gi)), ("m", m[:, 0]), ("logl", np.log(l)[:, 0])):
      out[name].append(val)
  return {n: np.stack(v) for n, v in out.items()}


def bounds(c, ref):
  """Per-element bound of every output (module docstring)."""
  lq, lk, dv = c.lq, c.lk, c.dv
  e = {"out": (TAU + gamma(2 * lk + 8)) * ref["A_out"], "dv": (TAU + gamma(lq + 8)) * ref["A_dv"],
       "dq": (TAU + gamma(lk + dv + 8)) * ref["A_dq"], "dk": (TAU + gamma(lq + dv + 8)) * ref["A_dk"],
       "lse": 8 * U * (np.abs(ref["m"]) + np.abs(ref["logl"])) + 8 * U + gamma(lk)}
  return {n: v + TINY for n, v in e.items()}


NAMES = {"out": ("image", "row", "col"), "lse": ("image", "row"), "dq": ("image", "row", "col"),
         "dk": ("image", "row", "col"), "dv": ("image", "row", "col")}
TAU_A = {"out": "A_out", "dq": "A_dq", "dk": "A_dk", "dv": "A_dv"}


def judge(c, got, ref, bnd, what):
  """The criterion on {output: values}; returns {output: worst err / (TAU A)} (lse: err / bound)."""
  ratios = {}
  for n, y in got.items():
    check_bound(y, ref[n], bnd[n], "%s %s" % (what, n), NAMES[n])
    err = np.abs(np.asarray(y, np.float64) - ref[n])
    scale = TAU * ref[TAU_A[n]] + TINY if n in TAU_A else bnd[n]
    ratios[n] = float(np.max(err / scale))
  return ratios


def run_attention(K, c, q, k, v, dout):
  """Forward and backward through the C-ABI on guarded buffers; returns ({output: values}, path and launch counts)."""
  lib = K.lib()
  b, lq, lk, dk, dv = c.batch, c.lq, c.lk, c.dk, c.dv
  ins = [Guarded(K, a) for a in (q, k, v, dout)]
  Q, Kb, V, DO = ins
  O, L = Guarded(K, np.full(b * lq * dv, SENTINEL, np.float32)), Guarded(K, np.full(b * lq, SENTINEL, np.float32))
  n0 = lib.launch_count()
  K._call("attention_fwd", Q.ptr, Kb.ptr, V.ptr, O.ptr, L.ptr, b, lq, lk, dk, dv)
  fwd = (_lib.PATH_NAMES[lib.get_option(_lib.OPT_LAST_PATH)], lib.launch_count() - n0)
  res = {}
  res["out"] = verify(O, np.arange(b * lq * dv).reshape(b, lq, dv), np.zeros((b, lq, dv), np.float32), c.id + " out",
                      NAMES["out"], (np.zeros((b, lq, dv)), np.full((b, lq, dv), np.inf)))[0]
  res["lse"] = verify(L, np.arange(b * lq).reshape(b, lq), np.zeros((b, lq), np.float32), c.id + " lse", NAMES["lse"],
                      (np.zeros((b, lq)), np.full((b, lq), np.inf)))[0]
  grads = {"dq": (b, lq, dk), "dk": (b, lk, dk), "dv": (b, lk, dv)}
  G = {n: Guarded(K, np.full(int(np.prod(s)), SENTINEL, np.float32)) for n, s in grads.items()}
  n0 = lib.launch_count()
  K._call("attention_bwd", Q.ptr, Kb.ptr, V.ptr, O.ptr, L.ptr, DO.ptr, G["dq"].ptr, G["dk"].ptr, G["dv"].ptr, b, lq, lk,
          dk, dv)
  bwd = (_lib.PATH_NAMES[lib.get_option(_lib.OPT_LAST_PATH)], lib.launch_count() - n0)
  for n, s in grads.items():        # only the output floats may change; the values are judged by the caller
    res[n] = verify(G[n], np.arange(int(np.prod(s))).reshape(s), np.zeros(s, np.float32), "%s %s" % (c.id, n),
                    NAMES[n], (np.zeros(s), np.full(s, np.inf)))[0]
  for buf, a, n in zip(ins + [O, L], (q, k, v, dout, res["out"], res["lse"]), ("q", "k", "v", "dout", "out", "lse")):
    verify(buf, np.arange(a.size).reshape(a.shape), a, "%s input %s after the backward" % (c.id, n), ("i",) * a.ndim)
  return res, fwd, bwd


def check_attention_case(K, c):
  q, k, v, dout, _ = draw(c)
  ref = reference64(q, k, v, dout)
  bnd = bounds(c, ref)
  first, fwd, bwd = run_attention(K, c, q, k, v, dout)
  assert_path(K, c.id + " forward", fwd[0], "tcgen05_tf32", fwd[1], 1)
  assert_path(K, c.id + " backward", bwd[0], "tcgen05_tf32", bwd[1], 3)
  ratios = judge(c, first, ref, bnd, c.id)
  second = run_attention(K, c, q, k, v, dout)[0]
  for n in first:
    assert np.array_equal(first[n].view(np.uint32), second[n].view(np.uint32)), "%s: two runs differ in %s" % (c.id, n)
  for n, r in ratios.items():
    record(K, n, r, c.id)
  return ratios


# misaligned twins: (entry point, operand, floats off): 2 floats keep 8-byte but break 16-byte alignment
MISALIGNED = [("fwd", "q", 2), ("fwd", "k", 1), ("fwd", "v", 2), ("fwd", "out", 1), ("fwd", "lse", 1),
              ("bwd", "q", 1), ("bwd", "k", 2), ("bwd", "v", 1), ("bwd", "dout", 2), ("bwd", "lse", 1),
              ("bwd", "dq", 1), ("bwd", "dk", 1), ("bwd", "dv", 1)]
MIS_CASE = C(1, 128, 128, 8, 32, "diffuse")


def check_misaligned(K, entry, operand, off):
  """The entry point refuses the pointer with CGAN_ERR_UNSUPPORTED naming the alignment, launches nothing and writes
  nothing (every buffer keeps its bits, guard bands included)."""
  c = MIS_CASE
  b, lq, lk, dk, dv = c.batch, c.lq, c.lk, c.dk, c.dv
  q, k, v, dout, _ = draw(c)
  vals = {"q": q, "k": k, "v": v, "dout": dout, "out": np.full((b, lq, dv), 0.5, np.float32),
          "lse": np.full((b, lq), 3.0, np.float32), "dq": np.full((b, lq, dk), SENTINEL, np.float32),
          "dk": np.full((b, lk, dk), SENTINEL, np.float32), "dv": np.full((b, lk, dv), SENTINEL, np.float32)}
  bufs = {n: Guarded(K, a, off if n == operand else 0) for n, a in vals.items()}
  p = {n: bf.ptr for n, bf in bufs.items()}
  lib = K.lib()
  n0 = lib.launch_count()
  with pytest.raises(_lib.CganError) as err:
    if entry == "fwd":
      K._call("attention_fwd", p["q"], p["k"], p["v"], p["out"], p["lse"], b, lq, lk, dk, dv)
    else:
      K._call("attention_bwd", p["q"], p["k"], p["v"], p["out"], p["lse"], p["dout"], p["dq"], p["dk"], p["dv"], b, lq,
              lk, dk, dv)
  msg = str(err.value)
  assert "failed (%d)" % 4 in msg and "aligned" in msg, msg                   # CGAN_ERR_UNSUPPORTED
  assert lib.launch_count() == n0, "%s with %s misaligned: %d kernels launched" % (entry, operand, lib.launch_count() - n0)
  for n, bf in bufs.items():
    got = bf.read()
    assert np.array_equal(got.view(np.uint32), bf.initial.view(np.uint32)), "%s: %s was written" % (entry, n)


# ---------------------------------------------------------------------------------------------------- softmax, rowdot

class Soft(object):
  """cgan_softmax_fwd / _bwd over rows x cols; misalign: every pointer 1-3 floats off 16 bytes; big: row offsets of
  +-1e4 with a spread of +-30 (and one row of one huge value among -1e30)."""

  def __init__(self, rows, cols, misalign=0, big=False):
    self.rows, self.cols, self.misalign, self.big = rows, cols, misalign, big

  @property
  def id(self):
    return "r%d-c%d%s%s" % (self.rows, self.cols, "-misaligned" if self.misalign else "", "-big" if self.big else "")

  @property
  def kernel(self):
    """The kernel cgan_softmax_fwd / _bwd pick (pointwise.cu)."""
    if not self.misalign and self.cols in (1024, 256):
      return "softmax warp%d" % (self.cols // 128)
    return "softmax block"


SOFTMAX_CASES = [
    Soft(37, 1), Soft(13, 3), Soft(101, 100), Soft(9, 255), Soft(1001, 256), Soft(1001, 256, misalign=1),
    Soft(7, 257), Soft(333, 1024), Soft(333, 1024, misalign=2), Soft(5, 1025), Soft(3, 4096), Soft(3, 4096, misalign=3),
    Soft(37, 1024, big=True), Soft(19, 256, big=True), Soft(11, 257, misalign=3, big=True),
]

ROWDOT_CASES = [(37, 1, 0), (9, 31, 0), (1001, 33, 0), (13, 100, 1), (333, 96, 0), (5, 1000, 2), (3, 4099, 0)]


def softmax_inputs(sc):
  rng = np.random.RandomState(seed_of(sc.id))
  x = (3.0 * rng.standard_normal((sc.rows, sc.cols))).astype(np.float32)
  if sc.big:
    x = (rng.uniform(-1e4, 1e4, (sc.rows, 1)) + 30.0 * rng.standard_normal((sc.rows, sc.cols))).astype(np.float32)
    x[0] = -1e30
    x[0, sc.cols // 2] = 1e30
  dy = rng.standard_normal((sc.rows, sc.cols)).astype(np.float32)
  return x, dy


def softmax_reference(x, y, dy):
  """(y64, bound) of the forward from x and (dx64, bound) of the backward from the float32 y and dy.
  forward: e = expf(x - m) carries u |x - m| (the rounded difference) + 4 u (expf, 2 ulp); the row sum gamma(cols) plus
  the e-weighted mean of its terms' errors; 1 / s and the product 2 u.  backward: the sum of cols products (gamma(cols)),
  the subtraction and the product."""
  x64 = x.astype(np.float64)
  m = x64.max(1, keepdims=True)
  e = np.exp(x64 - m)
  y64 = e / e.sum(1, keepdims=True)
  rel_e = U * np.abs(x64 - m) + 4 * U
  rel = rel_e + (y64 * rel_e).sum(1, keepdims=True) + gamma(x.shape[1] + 2) + 2 * U
  fwd = (y64, rel * y64 + TINY)
  p, g = y.astype(np.float64), dy.astype(np.float64)
  s, sa = (g * p).sum(1, keepdims=True), (np.abs(g) * p).sum(1, keepdims=True)
  bwd = (p * (g - s), gamma(x.shape[1] + 2) * p * (np.abs(g) + sa) + TINY)
  return fwd, bwd


def check_softmax_case(K, sc):
  x, dy = softmax_inputs(sc)
  rows, cols, mis = sc.rows, sc.cols, sc.misalign
  lib = K.lib()
  X, Y = Guarded(K, x, mis), Guarded(K, np.full(x.size, SENTINEL, np.float32), (2 * mis) % 4)
  offs = np.arange(x.size).reshape(rows, cols)
  n0 = lib.launch_count()
  K._call("softmax_fwd", Y.ptr, X.ptr, rows, cols)
  assert_path(K, sc.id + " fwd", "simt_fp32", "simt_fp32", lib.launch_count() - n0, 1)
  y = verify(Y, offs, np.zeros_like(x), sc.id + " softmax_fwd", ("row", "col"),
             (np.zeros(x.shape), np.full(x.shape, np.inf)))[0]
  verify(X, offs, x, sc.id + " softmax_fwd input", ("row", "col"))
  (y64, ey), (dx64, edx) = softmax_reference(x, y, dy)
  r1 = check_bound(y, y64, ey, sc.id + " softmax_fwd", ("row", "col"))
  DY, P = Guarded(K, dy, (3 * mis) % 4), Guarded(K, y, mis)
  DX = Guarded(K, np.full(x.size, SENTINEL, np.float32), (2 * mis) % 4)
  n0 = lib.launch_count()
  K._call("softmax_bwd", DX.ptr, DY.ptr, P.ptr, rows, cols)
  assert_path(K, sc.id + " bwd", "simt_fp32", "simt_fp32", lib.launch_count() - n0, 1)
  _, r2 = verify(DX, offs, np.zeros_like(x), sc.id + " softmax_bwd", ("row", "col"), (dx64, edx))
  record(K, sc.kernel, max(r1, r2), sc.id)
  return max(r1, r2)


def check_rowdot_case(K, rows, cols, mis):
  rng = np.random.RandomState(seed_of("rowdot-%d-%d" % (rows, cols)))
  a, b = rng.standard_normal((rows, cols)).astype(np.float32), rng.standard_normal((rows, cols)).astype(np.float32)
  A, B = Guarded(K, a, mis), Guarded(K, b, (mis + 1) % 4 if mis else 0)
  out = Guarded(K, np.full(rows, SENTINEL, np.float32), (2 * mis) % 4)
  lib = K.lib()
  n0 = lib.launch_count()
  K._call("rowdot", out.ptr, A.ptr, B.ptr, rows, cols)
  assert_path(K, "rowdot", "simt_fp32", "simt_fp32", lib.launch_count() - n0, 1)
  a64, b64 = a.astype(np.float64), b.astype(np.float64)
  # a lane adds every 32nd product (FMA chain), then a 5-level shuffle tree
  e = gamma(-(-cols // 32) + 6) * (np.abs(a64) * np.abs(b64)).sum(1) + TINY
  _, r = verify(out, np.arange(rows), np.zeros(rows, np.float32), "rowdot r%d-c%d" % (rows, cols), ("row",),
                ((a64 * b64).sum(1), e))
  record(K, "rowdot", r, "r%d-c%d" % (rows, cols))
  return r


# ---------------------------------------------------------------------------------------------------- GPU tests

@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  kernels.set_math_mode(1)
  yield kernels
  kernels.set_math_mode(0)


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_fused_attention_elementwise(K, c):
  check_attention_case(K, c)


@pytest.mark.gpu
@pytest.mark.parametrize("entry,operand,off", MISALIGNED, ids=["%s-%s+%d" % m for m in MISALIGNED])
def test_fused_attention_refuses_misaligned_operands(K, entry, operand, off):
  check_misaligned(K, entry, operand, off)


@pytest.mark.gpu
@pytest.mark.parametrize("sc", SOFTMAX_CASES, ids=[s.id for s in SOFTMAX_CASES])
def test_softmax_elementwise(K, sc):
  check_softmax_case(K, sc)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols,mis", ROWDOT_CASES, ids=["r%d-c%d%s" % (r, c, "-misaligned" if m else "")
                                                            for r, c, m in ROWDOT_CASES])
def test_rowdot_elementwise(K, rows, cols, mis):
  check_rowdot_case(K, rows, cols, mis)


# ---------------------------------------------------------------------------------------------------- CPU tests

def model_outputs(q, k, v, dout):
  out, lse = attention_tf32_model(q, k, v)
  dq, dk, dv = attention_tf32_model(q, k, v, dout=dout, out=out, lse=lse)
  return {"out": out, "lse": lse, "dq": dq, "dk": dk, "dv": dv}


def test_case_table_covers_the_kernel_branches():
  """Every NV instance (32, 64, 96, 128) of the three kernels at a padded and an unpadded dv, all eight dk, lq < lk,
  lq > lk, lq = lk = 128, BigGAN's two shapes, 1, 3 and a few hundred images, every regime; the routing designations
  cover every key position of the 64-key tiles; the operands keep every score and dP exact in fp32; each regime does
  what it claims (wide: flushed keys, offset: scores near -100, tied: exact ties)."""
  assert {16, 32, 48, 64, 80, 96, 112, 128} <= {c.dv for c in CASES}
  assert {nv_pad(c.dv) for c in CASES} == {32, 64, 96, 128}
  assert set(range(4, 33, 4)) <= {c.dk for c in CASES}
  assert any(c.lq < c.lk for c in CASES) and any(c.lq > c.lk for c in CASES)
  assert any(c.lq == c.lk == 128 for c in CASES)
  assert {(4096, 1024, 24, 96), (4096, 1024, 12, 48)} <= {(c.lq, c.lk, c.dk, c.dv) for c in CASES}
  assert {1, 3} <= {c.batch for c in CASES} and max(c.batch for c in CASES) >= 200
  assert {"diffuse", "wide", "offset", "tied", "routing"} == {c.regime for c in CASES}
  for c in CASES:
    if c.lq * c.lk > 2 ** 20:
      continue           # the BigGAN shapes: same generator, seconds of float64 here for no extra coverage
    q, k, v, dout, pi = draw(c)
    qa, ka = np.abs(q.astype(np.float64)), np.abs(k.astype(np.float64))
    unit = (1.0 / 16) ** 2 if c.regime == "wide" else (1.0 / 64) ** 2
    assert (qa @ ka.transpose(0, 2, 1)).max() / unit < 2 ** 24, c.id           # every partial sum of S is exact
    s = q.astype(np.float64) @ k.astype(np.float64).transpose(0, 2, 1)
    gap = s - s.max(2, keepdims=True)
    if c.regime == "routing":
      for pb in pi:
        assert len({int(j) % 64 for j in pb}) == 64 and len({int(j) // 64 for j in pb}) == c.lk // 64, c.id
        if c.lq >= c.lk:
          assert len(set(pb.tolist())) == c.lk, c.id
      top = np.take_along_axis(gap, pi[:, :, None], 2)
      assert (top == 0).all() and (np.sort(gap, 2)[:, :, -2] <= -4).all(), c.id    # pi(i) leads by well over 4
    if c.regime == "wide":
      assert (gap < -FLUSH).mean() > 0.05, c.id
    if c.regime == "offset":
      assert (s > -112).all() and (s < -88).all(), c.id
    if c.regime == "tied":
      assert (gap == 0).all(), c.id


def test_criterion_accepts_the_kernel_model_and_rejects_local_defects():
  """The kernels' arithmetic (attention_tf32_model, the contract in the attn_tc.cu header) passes the criterion on
  routing, wide and diffuse data; each local defect a kernel could have fails it at an element it names: two keys
  swapped inside one 64-key tile, one key tile dropped, rows r and r + 8 of lse swapped, a padded dv column read as
  non-zero, the last image read at a wrong stride."""
  route = C(3, 256, 512, 12, 48, "routing")
  for c in (route, C(2, 128, 256, 8, 80, "wide"), C(2, 256, 128, 20, 32, "diffuse")):
    q, k, v, dout, _ = draw(c)
    ref = reference64(q, k, v, dout)
    ratios = judge(c, model_outputs(q, k, v, dout), ref, bounds(c, ref), c.id + " model")
    assert max(ratios[n] for n in TAU_A) < 1.0, ratios

  q, k, v, dout, pi = draw(route)
  ref = reference64(q, k, v, dout)
  bnd = bounds(route, ref)

  def rejects(got, match, *outputs):
    for n in outputs:
      with pytest.raises(AssertionError, match=match):
        check_bound(got[n], ref[n], bnd[n], "defect " + n, NAMES[n])

  # two keys of image 1 inside key tile 2 swapped: in V only (P meets the wrong V row: a wrong load_t permutation or
  # register-fragment mapping), and in both K and V (the same attention over relabelled keys: O is unchanged, dK and
  # dV land on each other's rows)
  j1, j2 = sorted(int(j) for j in pi[1] if 128 <= j < 192)[:2]
  swap = lambda a: np.concatenate([a[:1], a[1:2][:, np.r_[0:j1, j2, j1 + 1:j2, j1, j2 + 1:a.shape[1]]], a[2:]])
  i = int(np.flatnonzero(pi[1] == j1)[0])
  got = model_outputs(q, k, swap(v), dout)
  rejects(got, r"image=1", "out")
  with pytest.raises(AssertionError):
    check_bound(got["out"][1, i], ref["out"][1, i], bnd["out"][1, i], "swapped key", ("col",))
  got = model_outputs(q, swap(k), swap(v), dout)
  check_bound(got["out"], ref["out"], bnd["out"], "relabelled keys", NAMES["out"])
  rejects(got, r"image=1, row=%d" % j1, "dk", "dv")
  # key tile 5 of image 0 dropped
  keep = np.r_[0:320, 384:512]
  o, _ = attention_tf32_model(q[:1], k[:1, keep], v[:1, keep])
  with pytest.raises(AssertionError, match=r"image=0"):
    check_bound(o, ref["out"][:1], bnd["out"][:1], "dropped tile", NAMES["out"])
  # rows 16 + r and 24 + r of lse swapped (the two rows one thread owns), on diffuse data where rows differ
  cd = C(1, 128, 128, 16, 32, "diffuse")
  qd, kd, vd, gd, _ = draw(cd)
  refd = reference64(qd, kd, vd, gd)
  lse = attention_tf32_model(qd, kd, vd)[1]
  lse[:, 16:24], lse[:, 24:32] = lse[:, 24:32].copy(), lse[:, 16:24].copy()
  with pytest.raises(AssertionError, match=r"image=0, row=1[6-9]|image=0, row=2"):
    check_bound(lse, refd["lse"], bounds(cd, refd)["lse"], "lse rows swapped", NAMES["lse"])
  # dv = 48 padded to 64 columns with the next row's values where the zero padding belongs (an unmasked load)
  def padded(a):
    flat = np.concatenate([a.ravel(), np.ones(16, np.float32)])
    rows = a.shape[0] * a.shape[1]
    idx = np.arange(rows)[:, None] * a.shape[2] + np.arange(64)[None, :]
    return flat[idx].reshape(a.shape[0], a.shape[1], 64)
  out, lse = attention_tf32_model(q, k, v)
  gq, gk, _ = attention_tf32_model(q, k, padded(v), dout=padded(dout), out=padded(out), lse=lse)
  rejects({"dq": gq, "dk": gk}, r"image=", "dq", "dk")
  # the last image of K and V read at image stride lq instead of lk
  kf, vf = k.reshape(-1, route.dk), v.reshape(-1, route.dv)
  last = (route.batch - 1) * route.lq
  kw, vw = k.copy(), v.copy()
  kw[-1], vw[-1] = kf[last:last + route.lk], vf[last:last + route.lk]
  got = model_outputs(q, kw, vw, dout)
  rejects(got, r"image=2", "out")
  assert np.array_equal(got["out"][:2], model_outputs(q, k, v, dout)["out"][:2])


def test_softmax_table_covers_the_kernels():
  kinds = {sc.kernel for sc in SOFTMAX_CASES}
  assert kinds == {"softmax warp8", "softmax warp2", "softmax block"}
  assert {1, 3, 100, 255, 256, 257, 1024, 1025, 4096} <= {sc.cols for sc in SOFTMAX_CASES}
  assert any(sc.misalign and sc.cols == 1024 for sc in SOFTMAX_CASES)
  assert any(sc.misalign and sc.cols == 256 for sc in SOFTMAX_CASES)
  assert any(sc.rows % 8 for sc in SOFTMAX_CASES if sc.kernel != "softmax block")
  assert any(cols % 32 for _, cols, _ in ROWDOT_CASES)


def test_softmax_criterion_rejects_one_misplaced_element():
  """The softmax bounds accept a float32 evaluation and reject a row normalised by a sum that lost one term."""
  sc = Soft(9, 255)
  x, dy = softmax_inputs(sc)
  x64 = x.astype(np.float64)
  e = np.exp((x - x.max(1, keepdims=True)).astype(np.float64)).astype(np.float32)
  y = (e * (np.float32(1) / e.sum(1, keepdims=True, dtype=np.float32))).astype(np.float32)
  (y64, ey), _ = softmax_reference(x, y, dy)
  check_bound(y, y64, ey, "fp32 softmax", ("row", "col"))
  j = int(np.argsort(x64[4])[-2])         # the second largest term of row 4 left out of its sum
  bad = y.copy()
  bad[4] = e[4] / (e[4].sum() - e[4, j])
  with pytest.raises(AssertionError, match="row=4"):
    check_bound(bad, y64, ey, "lost term", ("row", "col"))


def test_case_tables_on_the_emulator():
  """Every table through tests/abi_emulator.py: guard bands, layouts, the misaligned-pointer refusals and the references
  agree with the C-ABI's contract on the CPU (path and launch counts are the library's and not asserted here)."""
  from compare_gan_b200 import kernels
  with emulated_library():
    kernels.set_math_mode(1)
    for c in CASES:
      check_attention_case(kernels, c)
    for m in MISALIGNED:
      check_misaligned(kernels, *m)
    for sc in SOFTMAX_CASES:
      check_softmax_case(kernels, sc)
    for r in ROWDOT_CASES:
      check_rowdot_case(kernels, *r)
