"""The pointwise, pooling, loss, penalty and optimizer kernels of csrc/pointwise.cu and the tangent kernels of
csrc/jacobian.cu, element by element against float64.

Every GPU case keeps its inputs and outputs inside NaN-sentinel guard bands (tests/test_simt_exact_gpu.py, Guarded /
verify), asserts the number of kernels launched, and reports the first bad element decoded to its coordinates.  Where
a kernel has a float4 body (act_fwd / act_bwd, add_tf32, avgpool2, pool2d_fwd) the case has a misaligned twin: the same
operands 1-3 floats off 16-byte alignment, which run the scalar code and must give bit-identical results.

The verdict per element is one of two kinds.
  bit-exact  ops that round at most once: the float64 result rounded once to float32, or the numpy float32 operation
             where the kernel's single rounding is an fp32 product (copies, fills, one_hot, rot90, bias_add, ReLU and
             leaky ReLU both ways, add / add_tf32 with RNA TF32 rounding, max pools, avgpool2_bwd, globalpool_bwd,
             rowscale, scale_by_dev, argmax_one_hot, row_has_label, maxpool2_jvp, the hinge and Wasserstein gradients).
  bounded    |y - y64| <= e, with e = gamma(L) A + ulp terms + TINY: L the chain of dependent fp32 roundings (derived
             next to each kernel's reference below from its code), A the same computation over absolute values, the
             ulp terms the CUDA Math API maxima (expf 2 ulp, logf 1 ulp, log1pf 1 ulp, tanhf 2 ulp; the library is
             built without fast math), TINY = 2^-126 for results that leave the normal range.
The float64 references restate the reference's math (e.g. sigmoid_cross_entropy as max(x, 0) - x z + log1p(exp(-|x|)));
only the bounds know the kernels' arithmetic.

Leaky ReLU's gradient follows TF: tf.maximum(x, leak x) sends a tie's gradient to x, so d/dx = 1 where x >= 0 (-0
included) and leak elsewhere; ReLU's is [x > 0] (ReluGrad).

The CPU tests run every table through tests/abi_emulator.py and show that the criterion rejects injected local defects:
a shifted pool window, the real and fake gradients swapped, a loss mean over b - 1, Adam's bias correction one step off
and the old leaky tie rule.  The module prints, per kernel, its bit-exact case count and its worst err / bound."""
import math
import time

import numpy as np
import pytest

from tests.abi_emulator import emulated_library, relu_gate, rna_tf32
from tests.test_simt_exact_gpu import SENTINEL, Guarded, check_bound, emulated, gamma, seed_of, verify

U = 2.0 ** -24
TINY = 2.0 ** -126
EXPF, LOGF, LOG1PF, TANHF = 4 * U, 2 * U, 2 * U, 4 * U      # CUDA Math API maxima (2, 1, 1, 2 ulp) as relative errors
SMS = 132                                                 # H100 SXM; grid-stride sizes below exceed one sweep at any SM count <= 144
SWEEP = 4 * 144 * 16 * 256                                # floats one float4 grid sweep covers at 144 SMs
BLOCK_SUM = 10                                            # block_sum over 256 threads: 5 shuffle levels twice
SUMMARY = {}        # kernel -> {"exact": cases, "bound": cases, "worst": (err / bound, case)}


@pytest.fixture(scope="module", autouse=True)
def _report(pytestconfig):
  t0 = time.time()
  SUMMARY.clear()
  yield
  if not SUMMARY:
    return
  lines = ["pointwise kernels, %.1f s (bit-exact cases; bounded cases: worst err / bound):" % (time.time() - t0)]
  for k in sorted(SUMMARY):
    s = SUMMARY[k]
    txt = "  %-18s %3d bit-exact" % (k, s["exact"])
    if s["bound"]:
      txt += " %3d bounded, worst %.3e (%s)" % (s["bound"], s["worst"][0], s["worst"][1])
    lines.append(txt)
  capman = pytestconfig.pluginmanager.getplugin("capturemanager")
  tr = pytestconfig.pluginmanager.getplugin("terminalreporter")
  if capman is None or tr is None:
    print("\n".join(lines))
    return
  with capman.global_and_fixture_disabled():
    tr.ensure_newline()
    for line in lines:
      tr.write_line(line)


def record(K, kernel, case, ratio=None):
  if emulated(K):
    return
  s = SUMMARY.setdefault(kernel, {"exact": 0, "bound": 0, "worst": (0.0, "")})
  if ratio is None:
    s["exact"] += 1
  else:
    s["bound"] += 1
    if ratio >= s["worst"][0]:
      s["worst"] = (ratio, case)


def f32(a):
  return np.asarray(a, np.float32)


def d64(a):
  return np.asarray(a, np.float32).astype(np.float64)


def bits(*pattern):
  return np.array(pattern, np.uint32).view(np.float32)


def out_buf(K, n, mis=0):
  return Guarded(K, np.full(int(n), SENTINEL, np.float32), mis)


def launch(K, launches, entry, *args):
  """One C-ABI call; the library must launch exactly `launches` kernels (the emulator counts calls)."""
  lib = K.lib()
  n0 = lib.launch_count()
  K._call(entry, *args)
  if not emulated(K):
    assert lib.launch_count() - n0 == launches, "%s: %d kernels launched, expected %d" % (
        entry, lib.launch_count() - n0, launches)


def read(buf, shape, what, names, exact=None, bound=None):
  """The output of a guarded buffer, every other float unchanged: bit-exact against `exact`, or within bound = (y64,
  e).  Returns (values, worst err / bound or None)."""
  offs = np.arange(int(np.prod(shape))).reshape(shape)
  if exact is not None:
    return verify(buf, offs, f32(exact).reshape(shape), what, names)[0], None
  y64, e = bound
  return verify(buf, offs, f32(y64).reshape(shape), what, names, (np.reshape(y64, shape), np.reshape(e, shape)))


def unchanged(buf, a, what):
  verify(buf, np.arange(a.size), a, what + " (input)", ("i",))


def same_bits(a, b):
  return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


# ---------------------------------------------------------------------------------------------------- activations

ACT_NAMES = {1: "relu", 2: "lrelu", 3: "sigmoid", 4: "tanh01"}
ROUND = 0x100
LEAK = np.float32(0.2)
TIE = bits(0x3F801000, 0xBF801000, 0x40A01000, 0xC2481000, 0x3DCCF000)   # low 13 bits 0x1000: TF32 ties (RNA: away)


def special_inputs():
  """+-0, the leaky tie (x = +-0), logits at +-100, the exp overflow edges, TF32 rounding ties."""
  return np.concatenate([f32([0.0, -0.0, 100.0, -100.0, 1.0, -1.0, 88.0, -88.0, 89.0, -89.0, 1e-30, -1e-30, 0.5, -0.5]),
                         TIE, -TIE])


def act_operands(kind, n, salt=0):
  rng = np.random.RandomState(seed_of("act%d-%d" % (kind, n), salt))
  x = (3.0 * rng.standard_normal(n)).astype(np.float32)
  sp = special_inputs()
  x[:min(n, sp.size)] = sp[:n]
  g = rng.standard_normal(n).astype(np.float32)
  g[:min(n, TIE.size)] = TIE[:n]
  if kind in (1, 2):
    ref = x
  else:                               # the activation's output y in [0, 1], with its ends and midpoint
    ref = (1.0 / (1.0 + np.exp(-d64(x)))).astype(np.float32)
    ref[:min(n, 3)] = f32([0.0, 1.0, 0.5])[:n]
  return x, g, ref


def act_fwd_reference(kind, x, rnd):
  """(exact float32 or None, y64, e)."""
  x64 = d64(x)
  if kind == 1:
    y = np.maximum(x, np.float32(0))
    return (rna_tf32(y) if rnd else y), None, None
  if kind == 2:
    y = np.maximum(x, LEAK * x)                      # one rounding: the fp32 product leak * x
    return (rna_tf32(y) if rnd else y), None, None
  if kind == 3:
    with np.errstate(over="ignore"):
      y64 = 1.0 / (1.0 + np.exp(-x64))
    e = (EXPF + gamma(2)) * y64                      # expf, 1 + e, the reciprocal
  else:
    t = np.tanh(x64)
    y64 = (t + 1.0) / 2.0
    e = 0.5 * (TANHF * np.abs(t) + gamma(1) * (1.0 + np.abs(t)))   # tanhf, + 1 (the halving is exact)
  if rnd:
    e = e + 2.0 ** -11 * (y64 + e)                   # RNA to TF32: half a TF32 unit, 2^-11 relative
  return None, y64, e + TINY


def act_bwd_reference(kind, g, ref, leak, rnd):
  g64, r64 = d64(g), d64(ref)
  if kind == 1:
    y = np.where(ref > 0, g, np.float32(0))
    return (rna_tf32(y) if rnd else y), None, None
  if kind == 2:
    y = relu_gate(ref, g, leak)                      # TF's Maximum gradient: 1 where x >= 0, else the fp32 product leak * g
    return (rna_tf32(y) if rnd else y), None, None
  if kind == 3:                                      # g y (1 - y): 1 - y, two products
    y64 = g64 * r64 * (1.0 - r64)
    e = gamma(3) * np.abs(y64)
  else:                                              # g (1 - t^2) / 2, t = 2 y - 1: t, t^2, 1 - t^2 (cancels), the products
    t = 2.0 * r64 - 1.0
    y64 = g64 * 0.5 * (1.0 - t * t)
    e = gamma(5) * np.abs(g64) * 0.5 * (1.0 + t * t)
  if rnd:
    e = e + 2.0 ** -11 * (np.abs(y64) + e)
  return None, y64, e + TINY


class Vec(object):
  """act_fwd / act_bwd of one kind (op "act"), or add_tf32 (op "add", kind 0), over n floats; rnd: ACT_ROUND_TF32 /
  round_tf32; twin: rerun 1-3 floats off 16-byte alignment and demand the same bits."""

  def __init__(self, op, kind, n, rnd):
    self.op, self.kind, self.n, self.rnd = op, kind, n, rnd

  @property
  def id(self):
    name = ACT_NAMES[self.kind] if self.op == "act" else "add"
    return "%s-n%d%s" % (name, self.n, "-tf32" if self.rnd else "")

  @property
  def twin(self):
    return self.n >= 4


VEC_N = [1, 3, 4, 5, 1025, 1026, 1027, SWEEP + 4099]
VEC_CASES = ([Vec("act", k, n, r) for k in (1, 2, 3, 4) for r in (0, 1) for n in VEC_N] +
             [Vec("add", 0, n, r) for r in (0, 1) for n in VEC_N])


def run_act(K, vc, x, g, ref, mis):
  n, kind = vc.n, vc.kind | (ROUND if vc.rnd else 0)
  X, Y = Guarded(K, x, mis), out_buf(K, n, (2 * mis) % 4)
  launch(K, 1, "act_fwd", Y.ptr, X.ptr, kind, float(LEAK), n)
  DY, R, DX = Guarded(K, g, (3 * mis) % 4), Guarded(K, ref, mis), out_buf(K, n, (2 * mis) % 4)
  launch(K, 1, "act_bwd", DX.ptr, DY.ptr, R.ptr, kind, float(LEAK), n)
  for b, a, w in ((X, x, "x"), (DY, g, "dy"), (R, ref, "ref")):
    unchanged(b, a, "%s %s" % (vc.id, w))
  return Y, DX


def check_act_case(K, vc):
  x, g, ref = act_operands(vc.kind, vc.n)
  fx, fy64, fe = act_fwd_reference(vc.kind, x, vc.rnd)
  bx, by64, be = act_bwd_reference(vc.kind, g, ref, LEAK, vc.rnd)
  outs = []
  worst = 0.0
  for mis in ((0, 1 + vc.n % 3) if vc.twin else (0,)):
    Y, DX = run_act(K, vc, x, g, ref, mis)
    y, r1 = read(Y, (vc.n,), "%s act_fwd (misalign %d)" % (vc.id, mis), ("i",), fx, (fy64, fe))
    dx, r2 = read(DX, (vc.n,), "%s act_bwd (misalign %d)" % (vc.id, mis), ("i",), bx, (by64, be))
    outs.append((y, dx))
    worst = max(worst, r1 or 0.0, r2 or 0.0)
  if vc.twin:
    assert same_bits(outs[0][0], outs[1][0]) and same_bits(outs[0][1], outs[1][1]), \
        "%s: aligned and misaligned runs differ" % vc.id
  record(K, "act " + ACT_NAMES[vc.kind], vc.id, None if vc.kind in (1, 2) else worst)


def check_add_case(K, vc):
  rng = np.random.RandomState(seed_of(vc.id))
  a, b = rng.standard_normal(vc.n).astype(np.float32), rng.standard_normal(vc.n).astype(np.float32)
  sp = np.concatenate([TIE, -TIE, f32([1.0, -1.0])])
  a[:min(vc.n, sp.size)] = sp[:vc.n]                   # a + 0 = a: the tie reaches the rounding untouched
  b[:min(vc.n, sp.size)] = 0.0
  if vc.n > sp.size:
    a[sp.size - 2:sp.size], b[sp.size - 2:sp.size] = 1.0, -1.0    # x + (-x) = +0
  y = (a + b).astype(np.float32)                      # the float64 sum rounded once is the fp32 sum
  want = rna_tf32(y) if vc.rnd else y
  outs = []
  for mis in ((0, 1 + vc.n % 3) if vc.twin else (0,)):
    A, B, Y = Guarded(K, a, mis), Guarded(K, b, (3 * mis) % 4), out_buf(K, vc.n, (2 * mis) % 4)
    launch(K, 1, "add_tf32", Y.ptr, A.ptr, B.ptr, vc.n, vc.rnd)
    outs.append(read(Y, (vc.n,), "%s (misalign %d)" % (vc.id, mis), ("i",), want)[0])
  if vc.twin:
    assert same_bits(outs[0], outs[1]), "%s: aligned and misaligned runs differ" % vc.id
  record(K, "add_tf32", vc.id)


# ---------------------------------------------------------------------------------------------------- pools

class Pool(object):
  """avgpool2 / maxpool2 forward and backward over [n, h, w, c]; mis: operands 1-3 floats off 16 bytes (scalar kernels);
  ties: windows with four equal cells, two equal maxima and ReLU zeros (+0 and -0)."""

  def __init__(self, n, h, w, c, mis=0, ties=False):
    self.n, self.h, self.w, self.c, self.mis, self.ties = n, h, w, c, mis, ties

  @property
  def id(self):
    return "n%d-%dx%d-c%d%s%s" % (self.n, self.h, self.w, self.c, "-misaligned" if self.mis else "",
                                   "-ties" if self.ties else "")

  @property
  def vec4(self):
    return self.c % 4 == 0 and not self.mis


POOL_CASES = [Pool(3, 8, 8, 12), Pool(3, 8, 8, 12, mis=1), Pool(1, 2, 2, 4), Pool(1, 2, 2, 4, mis=3),
              Pool(2, 6, 10, 1), Pool(5, 4, 6, 3), Pool(3, 10, 4, 5, mis=2), Pool(3, 8, 6, 8, ties=True),
              Pool(2, 4, 4, 3, ties=True), Pool(1, 2, 2, 1, ties=True)]


def windows(x):
  """[n, h, w, c] -> [n, h/2, w/2, c, 4]: the four cells of each 2x2 window in row-major order."""
  n, h, w, c = x.shape
  return x.reshape(n, h // 2, 2, w // 2, 2, c).transpose(0, 1, 3, 5, 2, 4).reshape(n, h // 2, w // 2, c, 4)


def unwindows(wv, shape):
  n, h, w, c = shape
  return wv.reshape(n, h // 2, w // 2, c, 2, 2).transpose(0, 1, 4, 2, 5, 3).reshape(shape)


def tie_windows(rng, shape):
  """Integers with many ties: four equal cells, two equal maxima at every pair of positions, all-zero windows of +0 and
  -0 (a ReLU's output)."""
  x = rng.randint(-3, 4, size=shape).astype(np.float32)
  wv = windows(x).copy()
  flat = wv.reshape(-1, 4)
  for i in range(flat.shape[0]):
    kind = i % 5
    if kind == 0:
      flat[i] = 2.0
    elif kind == 1:
      a, b = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)][(i // 5) % 6]
      flat[i] = -1.0
      flat[i, a] = flat[i, b] = 3.0
    elif kind == 2:
      flat[i] = f32([0.0, -0.0, 0.0, -0.0])[np.roll(np.arange(4), i // 5)]
  return unwindows(wv, shape)


def pool_operands(pc):
  rng = np.random.RandomState(seed_of(pc.id))
  shape = (pc.n, pc.h, pc.w, pc.c)
  x = tie_windows(rng, shape) if pc.ties else rng.standard_normal(shape).astype(np.float32)
  g = rng.standard_normal((pc.n, pc.h // 2, pc.w // 2, pc.c)).astype(np.float32)
  return x, g


def first_max(wv):
  """Index of the first maximum of each window (row-major), as TF's MaxPoolGrad routes the gradient."""
  return np.argmax(d64(wv), axis=-1)


def pool_reference(x, g):
  wv = windows(x)
  x64 = d64(wv)
  avg64 = x64.mean(-1)
  avg_e = gamma(3) * np.abs(x64).mean(-1) + TINY             # three sums (the quarter is exact)
  mx = wv.max(-1)
  arg = first_max(wv)
  dmax = np.zeros(wv.shape, np.float32)
  np.put_along_axis(dmax, arg[..., None], g[..., None], -1)
  davg = np.repeat((np.float32(0.25) * g)[..., None], 4, -1)   # exact: a quarter of g
  return {"avg": (avg64, avg_e), "max": mx, "dmax": unwindows(dmax, x.shape), "davg": unwindows(davg, x.shape)}


def check_pool_case(K, pc, mis=None):
  mis = pc.mis if mis is None else mis
  x, g = pool_operands(pc)
  ref = pool_reference(x, g)
  shape, oshape = x.shape, g.shape
  args = (pc.n, pc.h, pc.w, pc.c)
  names = ("n", "y", "x", "c")
  X, G = Guarded(K, x, mis), Guarded(K, g, (2 * mis) % 4)
  res = {}
  for name, entry, ins, osh in (("avg", "avgpool2_fwd", (X,), oshape), ("max", "maxpool2_fwd", (X,), oshape),
                                ("davg", "avgpool2_bwd", (G,), shape), ("dmax", "maxpool2_bwd", (G, X), shape)):
    Y = out_buf(K, int(np.prod(osh)), (3 * mis) % 4)
    launch(K, 1, entry, Y.ptr, *[b.ptr for b in ins], *args)
    if name == "avg":
      res[name], r = read(Y, osh, pc.id + " " + entry, names, bound=ref["avg"])
      record(K, "avgpool2_fwd", pc.id, r)
    else:
      res[name] = read(Y, osh, pc.id + " " + entry, names, exact=ref[name])[0]
      record(K, entry, pc.id)
  unchanged(X, x, pc.id + " x")
  unchanged(G, g, pc.id + " dy")
  return res


def check_pool_twin(K, pc):
  """The float4 kernels (aligned, c % 4 == 0) and the scalar ones (the same operands 1 float off) give the same bits."""
  a = check_pool_case(K, pc)
  b = check_pool_case(K, pc, mis=1)
  for k in a:
    assert same_bits(a[k], b[k]), "%s: %s differs between the float4 and the scalar kernel" % (pc.id, k)


class Pool2d(object):
  """pool2d_fwd (Inception's pools): k 3, stride s, SAME or VALID, max (mode 0) or avg (mode 1, padded cells excluded
  from the divisor) over [2, hw, hw, c]."""

  def __init__(self, hw, stride, pad, mode, c):
    self.hw, self.stride, self.pad, self.mode, self.c = hw, stride, pad, mode, c

  @property
  def id(self):
    return "%s-%d-s%d-%s-c%d" % ("max" if self.mode == 0 else "avg", self.hw, self.stride, self.pad, self.c)

  def geometry(self):
    """(oh, pad_t): TF's SAME (out = ceil(h / s), the odd cell of padding at the bottom) or VALID."""
    h, s, k = self.hw, self.stride, 3
    if self.pad == "SAME":
      oh = -(-h // s)
      return oh, max((oh - 1) * s + k - h, 0) // 2
    return (h - k) // s + 1, 0


POOL2D_CASES = [Pool2d(hw, s, p, m, c) for hw in (35, 17, 8) for s in (1, 2) for p in ("SAME", "VALID")
                for m in (0, 1) for c in (8, 3)]


def pool2d_reference(pc, x):
  n, h, w, c = x.shape
  oh, pt = pc.geometry()
  x64 = d64(x)
  y64 = np.zeros((n, oh, oh, c))
  a64 = np.zeros((n, oh, oh, c))
  cnt = np.zeros((oh, oh))
  for i in range(oh):
    for j in range(oh):
      r0, c0 = i * pc.stride - pt, j * pc.stride - pt
      rs, cs = slice(max(r0, 0), min(r0 + 3, h)), slice(max(c0, 0), min(c0 + 3, w))
      win = x64[:, rs, cs, :]
      cnt[i, j] = win.shape[1] * win.shape[2]
      y64[:, i, j] = win.max((1, 2)) if pc.mode == 0 else win.mean((1, 2))
      a64[:, i, j] = np.abs(win).mean((1, 2))
  if pc.mode == 0:
    return y64.astype(np.float32), None
  return y64, gamma(cnt[None, :, :, None]) * a64 + TINY      # cnt - 1 sums and the correctly rounded division


def check_pool2d_case(K, pc, mis=0):
  rng = np.random.RandomState(seed_of(pc.id))
  n, hw, c = 2, pc.hw, pc.c
  x = rng.standard_normal((n, hw, hw, c)).astype(np.float32)
  if pc.mode == 0:
    x[0, :4, :4, 0] = 1.5                                 # tied maxima
  oh, pt = pc.geometry()
  exact, e = pool2d_reference(pc, x)
  X, Y = Guarded(K, x, mis), out_buf(K, n * oh * oh * c, (2 * mis) % 4)
  launch(K, 1, "pool2d_fwd", Y.ptr, X.ptr, n, hw, hw, c, 3, pc.stride, pt, pt, oh, oh, pc.mode)
  what = "%s pool2d%s" % (pc.id, " (misaligned %d)" % mis if mis else "")
  if pc.mode == 0:
    y, r = read(Y, (n, oh, oh, c), what, ("n", "y", "x", "c"), exact=exact)
  else:
    y, r = read(Y, (n, oh, oh, c), what, ("n", "y", "x", "c"), bound=(exact, e))
  unchanged(X, x, what)
  record(K, "pool2d %s" % ("max" if pc.mode == 0 else "avg"), pc.id, r)
  return y


def check_pool2d(K, pc):
  y = check_pool2d_case(K, pc)
  if pc.c % 4 == 0:                                      # the float4 kernel's misaligned twin: the scalar kernel
    y2 = check_pool2d_case(K, pc, mis=1 + pc.hw % 3)
    assert same_bits(y, y2), "%s: the float4 and the scalar pool2d kernels differ" % pc.id


GLOBAL_CASES = [(3, hw, c, mean) for hw in (1, 9, 36, 64) for c in (5, 16) for mean in (True, False)]


def check_globalpool(K, n, hw, c, mean):
  cid = "n%d-hw%d-c%d-%s" % (n, hw, c, "mean" if mean else "sum")
  rng = np.random.RandomState(seed_of(cid))
  x, g = rng.standard_normal((n, hw, c)).astype(np.float32), rng.standard_normal((n, c)).astype(np.float32)
  scale = np.float32(1.0 / hw) if mean else np.float32(1.0)
  X, Y = Guarded(K, x), out_buf(K, n * c)
  launch(K, 1, "globalpool_fwd", Y.ptr, X.ptr, n, hw, c, float(scale))
  div = hw if mean else 1
  # hw - 1 sums, the product with the rounded scale (whose own rounding, for 1 / hw, is one more u)
  y64, e = d64(x).sum(1) / div, gamma(hw + 1) * np.abs(d64(x)).sum(1) / div + TINY
  _, r = read(Y, (n, c), cid + " globalpool_fwd", ("n", "c"), bound=(y64, e))
  record(K, "globalpool_fwd", cid, r)
  G, DX = Guarded(K, g), out_buf(K, n * hw * c)
  launch(K, 1, "globalpool_bwd", DX.ptr, G.ptr, n, hw, c, float(scale))
  read(DX, (n, hw, c), cid + " globalpool_bwd", ("n", "hw", "c"), exact=np.repeat((scale * g)[:, None], hw, 1))
  record(K, "globalpool_bwd", cid)


# ---------------------------------------------------------------------------------------------------- losses

LOSS_NAMES = {0: "non_saturating", 1: "hinge", 2: "wasserstein", 3: "least_squares"}
LOSS_B = [1, 37, 256, 257, 1000, 4096]
LOSS_CASES = [(k, which, b) for k in (0, 1, 2, 3) for which in (0, 1) for b in LOSS_B]


def logits(b, salt):
  """N(0, 3) logits with the edges: +-100, the expf overflow edges, hinge's kinks at exactly +-1, +-0."""
  rng = np.random.RandomState(seed_of("logits-%d" % b, salt))
  z = (3.0 * rng.standard_normal(b)).astype(np.float32)
  sp = f32([1.0, -1.0, 100.0, -100.0, 0.0, -0.0, 89.0, -89.0, 20.0, -20.0, 1.0, -1.0])
  sp = np.roll(sp, salt)
  z[:min(b, sp.size)] = sp[:b]
  return z


def sig64(x):
  with np.errstate(over="ignore"):
    return 1.0 / (1.0 + np.exp(-x))


def loss_reference(kind, which, r, f):
  """The reference's losses (gans/loss_lib.py) and gradients in float64 with their bounds:
  {"out4": (y64, e), "dl": (y64, e)}.  Sums: ceil(b / 256) terms per thread, then block_sum; the means multiply by the
  rounded 1 / b; a term's own error is bounded per kernel below."""
  b = r.size
  r64, f64 = d64(r), d64(f)
  L = -(-b // 256) + BLOCK_SUM + 3                      # the sum, the rounded 1 / b, the product, d = a + c
  if kind == 0:
    sce = lambda x, z: np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))
    # sce: max(x, 0) - x z (one rounding), log1pf(expf(-|x|)) (the expf error shrinks through log1p), the sum
    term_a = lambda x: np.abs(np.maximum(x, 0) - x) + np.abs(x) + np.log1p(np.exp(-np.abs(x)))
    te = lambda x: (gamma(2) + EXPF + LOG1PF) * term_a(x)
    terms = (sce(r64, 1.0), sce(f64, 0.0), sce(f64, 1.0))
    absd = (term_a(r64), term_a(f64), term_a(f64))
    terr = (te(r64), te(f64), te(f64))
  elif kind == 1:
    terms = (np.maximum(1.0 - r64, 0), np.maximum(1.0 + f64, 0), -f64)
    absd = (1.0 + np.abs(r64), 1.0 + np.abs(f64), np.abs(f64))
    terr = (U * absd[0], U * absd[1], 0 * f64)
  elif kind == 2:
    terms = (-r64, f64, -f64)
    absd = (np.abs(r64), np.abs(f64), np.abs(f64))
    terr = (0 * r64, 0 * f64, 0 * f64)
  else:
    pr, pf = sig64(r64), sig64(f64)
    terms = ((pr - 1.0) ** 2, pf ** 2, 0.5 * (pf - 1.0) ** 2)
    # p = 1 / (1 + expf(-x)) carries EXPF + 2u relative: at most 7u absolute, so (p - 1)^2 and p^2 at most 16u + gamma(2)
    absd = (np.ones(b), np.ones(b), 0.5 * np.ones(b))
    terr = tuple(gamma(20) * a for a in absd)
  sums = [t.sum() / b for t in terms]
  errs = [(te_.sum() + gamma(L) * a.sum()) / b for te_, a in zip(terr, absd)]
  d = sums[0] + sums[1]
  de = errs[0] + errs[1] + U * (abs(sums[0]) + abs(sums[1]))
  if kind == 3:
    d, de = 0.5 * d, 0.5 * de
  out4 = (np.array([d, sums[0], sums[1], sums[2]]), np.array([de, errs[0], errs[1], errs[2]]) + TINY)
  # gradients w.r.t. [real; fake]
  zero = np.zeros(b)
  if kind == 0:
    pr, pf = sig64(r64), sig64(f64)
    # (p - 1) / b: p to 6u relative (7u absolute), the subtraction, the product with the rounded 1 / b
    if which == 0:
      dl = np.concatenate([(pr - 1.0) / b, pf / b])
    else:
      dl = np.concatenate([zero, (pf - 1.0) / b])
    e = np.concatenate([zero if which else gamma(10) / b + zero, gamma(10) * (pf if which == 0 else 1.0 + zero) / b])
  elif kind == 1:                                        # exact: +-1/b rounded once, or 0; ReluGrad's 0 at the kinks
    if which == 0:
      dl = np.concatenate([np.where(1.0 - r64 > 0, -1.0 / b, 0.0), np.where(1.0 + f64 > 0, 1.0 / b, 0.0)])
    else:
      dl = np.concatenate([zero, -1.0 / b + zero])
    e = np.zeros(2 * b)
  elif kind == 2:
    dl = np.concatenate([zero - (0 if which else 1.0 / b), (-1.0 if which else 1.0) / b + zero])
    e = np.zeros(2 * b)
  else:
    pr, pf = sig64(r64), sig64(f64)
    # products of p (6u relative) and q = 1 - p, which carries p's error as 8u ABSOLUTE (p rounds to 1 for x > 17):
    # p q^2 within p ((q + 8u)^2 (1 + gamma(20)) - q^2), p^2 q within p^2 ((q + 8u)(1 + gamma(20)) - q)
    e_pq2 = lambda p: p * ((np.abs(1.0 - p) + 8 * U) ** 2 * (1 + gamma(20)) - (1.0 - p) ** 2) / b
    e_p2q = lambda p: p * p * ((np.abs(1.0 - p) + 8 * U) * (1 + gamma(20)) - np.abs(1.0 - p)) / b
    if which == 0:
      dl = np.concatenate([(pr - 1.0) * pr * (1.0 - pr) / b, pf * pf * (1.0 - pf) / b])
      e = np.concatenate([e_pq2(pr), e_p2q(pf)])
    else:
      dl = np.concatenate([zero, (pf - 1.0) * pf * (1.0 - pf) / b])
      e = np.concatenate([zero, e_pq2(pf)])
  if kind in (1, 2):                                     # bit-exact: the float64 gradient rounded once
    return {"out4": out4, "dl": (dl.astype(np.float32).astype(np.float64), e)}
  return {"out4": out4, "dl": (dl, e + TINY)}


def loss_id(kind, which, b):
  return "%s-%s-b%d" % (LOSS_NAMES[kind], "d" if which == 0 else "g", b)


def judge_loss(cid, ref, out4, dl):
  r1 = check_bound(out4, ref["out4"][0], ref["out4"][1], cid + " out4", ("output",))
  r2 = check_bound(dl.reshape(2, -1), ref["dl"][0].reshape(2, -1), ref["dl"][1].reshape(2, -1), cid + " dlogits",
                   ("half (0 real, 1 fake)", "i"))
  return max(r1, r2)


def check_loss_case(K, kind, which, b):
  cid = loss_id(kind, which, b)
  r, f = logits(b, 0), logits(b, 5)
  ref = loss_reference(kind, which, r, f)
  R, F, O, D = Guarded(K, r), Guarded(K, f), out_buf(K, 4), out_buf(K, 2 * b)
  launch(K, 1, "gan_loss", kind, R.ptr, F.ptr, b, O.ptr, D.ptr, which)
  out4 = read(O, (4,), cid + " out4", ("output",), bound=ref["out4"])[0]
  dl = read(D, (2 * b,), cid + " dlogits", ("i",), bound=ref["dl"])[0]
  unchanged(R, r, cid + " real")
  unchanged(F, f, cid + " fake")
  record(K, "gan_loss " + LOSS_NAMES[kind], cid, judge_loss(cid, ref, out4, dl))


# ---------------------------------------------------------------------------------------------------- gp_penalty

GP_CASES = [(1, 1), (1, 1000), (5, 1000), (5, 3 * 128 * 128), (256, 3 * 32 * 32), (256, 1)]
GP_WEIGHT = np.float32(10.0)


def gp_operands(n, per):
  """N(0, 1 / per) rows (slopes near 1); row 0 has a slope a few ulp from 1 (s - 1 cancels), row 1 (n > 1) is all
  zero (slope sqrt(1e-4) = 0.01)."""
  rng = np.random.RandomState(seed_of("gp-%d-%d" % (n, per)))
  g = (rng.standard_normal((n, per)) / math.sqrt(per)).astype(np.float32)
  g[0] = 0.0
  g[0, 0] = np.float32(math.sqrt(1.0 - 1e-4)) + np.float32(3 * 2.0 ** -24)
  if n > 1:
    g[1] = 0.0
  return g


def gp_reference(g, weight):
  """slope = sqrt(1e-4 + sum g^2), pen = mean((slope - 1)^2), dg = weight 2 / n (slope - 1) / slope g, with bounds:
  the slope's sum has ceil(per / 256) + block_sum roundings plus 1e-4 rounded to fp32 and the correctly rounded sqrtf,
  so s carries es = s (gamma(Ls) + 2u); d = s - 1 then es + u |d|."""
  n, per = g.shape
  g64 = d64(g)
  ss = (g64 * g64).sum(1)
  s = np.sqrt(1e-4 + ss)
  d = s - 1.0
  es = s * (gamma(-(-per // 256) + BLOCK_SUM + 2) + 2 * U)
  ed = es + U * np.abs(d)
  Ln = -(-n // 256) + BLOCK_SUM + 2
  pen = (d * d).mean()
  pe = (2 * np.abs(d) * ed + ed * ed).mean() + gamma(Ln) * (d * d).mean() + TINY
  coef = 2.0 * float(weight) / n
  dg = coef * (d / s)[:, None] * g64
  dge = coef * np.abs(g64) / s[:, None] * (ed + np.abs(d) * (gamma(4) + es / s))[:, None] + TINY
  return (np.array([pen]), np.array([pe])), (dg, dge)


def check_gp_case(K, n, per):
  cid = "n%d-per%d" % (n, per)
  g = gp_operands(n, per)
  (pen64, pe), (dg64, dge) = gp_reference(g, GP_WEIGHT)
  G, P, DG = Guarded(K, g), out_buf(K, 1), out_buf(K, n * per)
  launch(K, 3, "gp_penalty", P.ptr, DG.ptr, G.ptr, n, per, float(GP_WEIGHT))
  _, r1 = read(P, (1,), cid + " penalty", ("i",), bound=(pen64, pe))
  _, r2 = read(DG, (n, per), cid + " dg", ("sample", "i"), bound=(dg64, dge))
  unchanged(G, g, cid + " g")
  P2 = out_buf(K, 1)                                     # without dg: the penalty alone, two launches
  launch(K, 2, "gp_penalty", P2.ptr, None, G.ptr, n, per, float(GP_WEIGHT))
  read(P2, (1,), cid + " penalty without dg", ("i",), bound=(pen64, pe))
  record(K, "gp_penalty", cid, max(r1, r2))


# ---------------------------------------------------------------------------------------------------- SSGAN / S3GAN

ROT_ROWS = [4, 256, 260, 1024]
XENT_CASES = [(rows, w) for rows in (4, 255, 256, 257, 1024) for w in ("none", "zeros")] + [(257, "all-zero")]


def rotation_reference(z):
  """-mean_r log(softmax(z_r)[r / m] + 1e-10) and its gradient, with bounds.  Per row: den sums 4 expf(z - mx) (each
  u |z - mx| + EXPF), p_y = expf / den, logf(p_y + eps); the row terms are summed (rows / 256 + block_sum)."""
  rows, nrot = z.shape
  z64 = d64(z)
  lab = np.arange(rows) // (rows // nrot)
  mx = z64.max(1, keepdims=True)
  e = np.exp(z64 - mx)
  p = e / e.sum(1, keepdims=True)
  py = p[np.arange(rows), lab]
  lr = -np.log(py + 1e-10)
  rel = 2 * (U * np.abs(z64 - mx).max(1) + EXPF) + gamma(nrot + 3)
  L = -(-rows // 256) + BLOCK_SUM + 1
  loss = lr.mean()
  le = (rel + U + LOGF * np.abs(lr)).mean() + gamma(L) * np.abs(lr).mean() + TINY
  onehot = np.zeros_like(p)
  onehot[np.arange(rows), lab] = 1.0
  coef = -(py / (py + 1e-10)) / rows
  dz = coef[:, None] * (onehot - p)
  relp = rel[:, None] + U * np.abs(z64 - mx) + EXPF
  dze = np.abs(coef)[:, None] * (np.abs(onehot - p) * (relp + gamma(6)) + relp * p) + TINY
  return (np.array([loss]), np.array([le])), (dz, dze)


def check_rotation_case(K, rows):
  cid = "rotation-r%d" % rows
  rng = np.random.RandomState(seed_of(cid))
  z = (2.0 * rng.standard_normal((rows, 4))).astype(np.float32)
  z[0] = [30.0, -30.0, 0.0, 0.0]                        # a confident row
  z[-1] = [-40.0, 40.0, 40.0, 40.0]                      # a label with p ~ e^-80: the 1e-10 floor of the log
  (l64, le), (dz64, dze) = rotation_reference(z)
  Z, L, D = Guarded(K, z), out_buf(K, 1), out_buf(K, rows * 4)
  launch(K, 1, "rotation_loss", L.ptr, D.ptr, Z.ptr, rows, 4)
  _, r1 = read(L, (1,), cid + " loss", ("i",), bound=(l64, le))
  _, r2 = read(D, (rows, 4), cid + " dlogits", ("row", "col"), bound=(dz64, dze))
  unchanged(Z, z, cid)
  record(K, "rotation_loss", cid, max(r1, r2))


def xent_operands(rows, wkind, cols=10):
  rng = np.random.RandomState(seed_of("xent-%d-%s" % (rows, wkind)))
  z = (2.0 * rng.standard_normal((rows, cols))).astype(np.float32)
  lab = rng.dirichlet(np.ones(cols), rows).astype(np.float32)             # soft labels
  lab[::3] = np.eye(cols, dtype=np.float32)[rng.randint(0, cols, rows)][::3]   # one-hot rows
  lab[1::7] = 0.0                                                           # unlabelled rows
  w = None
  if wkind == "zeros":
    w = rng.uniform(0.5, 2.0, rows).astype(np.float32)
    w[::4] = 0.0
  elif wkind == "all-zero":
    w = np.zeros(rows, np.float32)
  return z, lab, w


def xent_reference(z, lab, w):
  """sum_r w_r ce_r / #{w_r != 0} (0 when no weight is non-zero), ce_r = -sum_j l_j log softmax(z_r)_j, and d/dz.
  Bounds from the kernel's per-row chain: den (cols expf of rounded differences), logf(den), lsum, the dot of l with
  z - mx (cols products), w (lsum lden - dot), the row sum over threads and block_sum, the product with 1 / present."""
  rows, cols = z.shape
  z64, l64 = d64(z), d64(lab)
  w64 = np.ones(rows) if w is None else d64(w)
  mx = z64.max(1, keepdims=True)
  e = np.exp(z64 - mx)
  den = e.sum(1, keepdims=True)
  lden = np.log(den)
  ce = -(l64 * (z64 - mx - lden)).sum(1)
  present = float((w64 != 0).sum())
  inv = 1.0 / present if present > 0 else 0.0
  loss = (w64 * ce).sum() * inv
  lsum = l64.sum(1)
  D = (l64 * np.abs(z64 - mx)).sum(1)
  rel_den = U * np.abs(z64 - mx).max(1) + EXPF + gamma(cols)
  row_e = np.abs(w64) * (lsum * (rel_den + LOGF * np.abs(lden[:, 0])) + gamma(cols + 2) * (lsum * np.abs(lden[:, 0]) + D)
                         + gamma(3) * (lsum * np.abs(lden[:, 0]) + D))
  L = -(-rows // 256) + BLOCK_SUM + 2
  A = (np.abs(w64) * (lsum * np.abs(lden[:, 0]) + D)).sum()
  le = (row_e.sum() + gamma(L) * A) * inv + TINY
  p = e / den
  dz = (w64 * inv)[:, None] * (lsum[:, None] * p - l64)
  relp = rel_den[:, None] + U * np.abs(z64 - mx) + EXPF + gamma(4)
  dze = (np.abs(w64) * inv)[:, None] * (lsum[:, None] * p * relp + gamma(4) * np.abs(lsum[:, None] * p - l64)) + TINY
  return (np.array([loss]), np.array([le])), (dz, dze)


def check_xent_case(K, rows, wkind):
  cid = "xent-r%d-w%s" % (rows, wkind)
  z, lab, w = xent_operands(rows, wkind)
  cols = z.shape[1]
  (l64, le), (dz64, dze) = xent_reference(z, lab, w)
  Z, LB, L, D = Guarded(K, z), Guarded(K, lab), out_buf(K, 1), out_buf(K, rows * cols)
  W = Guarded(K, w) if w is not None else None
  launch(K, 1, "softmax_xent", L.ptr, D.ptr, Z.ptr, LB.ptr, W.ptr if W else None, rows, cols)
  _, r1 = read(L, (1,), cid + " loss", ("i",), bound=(l64, le))
  _, r2 = read(D, (rows, cols), cid + " dlogits", ("row", "col"), bound=(dz64, dze))
  if wkind == "all-zero":                               # no example counts: loss and gradient exactly 0
    read(L, (1,), cid + " loss", ("i",), exact=np.zeros(1))
    read(D, (rows, cols), cid + " dlogits", ("row", "col"), exact=np.zeros((rows, cols)))
  record(K, "softmax_xent", cid, max(r1, r2))


def check_heads(K):
  """argmax_one_hot with ties (the first index wins), row_has_label on exact label sums, rot90 k = 1, 2, 3."""
  rng = np.random.RandomState(seed_of("heads"))
  rows, cols = 300, 10
  z = rng.randint(-2, 3, size=(rows, cols)).astype(np.float32)     # many tied maxima
  z[0] = 1.0
  z[1] = -0.0
  z[1, 5] = 0.0
  Z, O = Guarded(K, z), out_buf(K, rows * cols)
  launch(K, 1, "argmax_one_hot", O.ptr, Z.ptr, rows, cols)
  read(O, (rows, cols), "argmax_one_hot", ("row", "col"), exact=np.eye(cols, dtype=np.float32)[np.argmax(d64(z), 1)])
  record(K, "argmax_one_hot", "r%d-c%d" % (rows, cols))
  y = np.zeros((rows, cols), np.float32)
  y[::2, 3] = 1.0
  y[1::6, :4] = 0.125                                    # sum 0.5: not a label
  y[3::6, :5] = 0.125                                    # sum 0.625
  Y, O = Guarded(K, y), out_buf(K, rows)
  launch(K, 1, "row_has_label", O.ptr, Y.ptr, rows, cols)
  read(O, (rows,), "row_has_label", ("row",), exact=(d64(y).sum(1) > 0.5).astype(np.float32))
  record(K, "row_has_label", "r%d-c%d" % (rows, cols))
  for k in (1, 2, 3):
    for c in (1, 3):
      x = rng.standard_normal((3, 7, 7, c)).astype(np.float32)
      X, O = Guarded(K, x), out_buf(K, x.size)
      launch(K, 1, "rot90", O.ptr, X.ptr, 3, 7, c, k)
      read(O, x.shape, "rot90 k%d c%d" % (k, c), ("n", "y", "x", "c"), exact=np.rot90(x, k, axes=(1, 2)))
      record(K, "rot90", "k%d-c%d" % (k, c))


# ---------------------------------------------------------------------------------------------------- Adam + EMA

class Adam(object):
  def __init__(self, n, t, gscale, ema_on):
    self.n, self.t, self.gscale, self.ema_on = n, t, gscale, ema_on

  @property
  def id(self):
    return "n%d-t%d-gs%g-ema%s" % (self.n, self.t, self.gscale, "on" if self.ema_on else "off")


ADAM_CASES = [Adam(1000, 1, 0.25, False), Adam(1000, 1, 0.25, True), Adam(1000, 2, 1.0 / 3, True),
              Adam(1000, 2, 1.0 / 3, False), Adam(1000, 1000, 0.5, True), Adam(1000, 10 ** 6, 0.25, True),
              Adam(SWEEP // 4 + 777, 1000, 0.5, False), Adam(SWEEP // 4 + 777, 3, 0.25, True)]
ADAM_HP = dict(lr=np.float32(2e-4), b1=np.float32(0.5), b2=np.float32(0.999), eps=np.float32(1e-8),
               decay=np.float32(0.9999))


def adam_state(ac):
  rng = np.random.RandomState(seed_of(ac.id))
  n = ac.n
  p = rng.standard_normal(n).astype(np.float32)
  g = rng.standard_normal(n).astype(np.float32)
  m = (0.1 * rng.standard_normal(n)).astype(np.float32)
  v = (1e-2 * rng.standard_normal(n) ** 2).astype(np.float32)
  ema = (p + 0.01 * rng.standard_normal(n)).astype(np.float32)
  g[:3], v[:3], m[:3] = 0.0, 0.0, 0.0                   # sqrt(0) + eps
  return p, g, m, v, ema


def adam_reference(ac, p, g, m, v, ema, t):
  """One Adam + EMA step in float64 from the fp32 state (tf.train.AdamOptimizer, ExponentialMovingAverage) with the
  fp32 hyper-parameters, and per-element bounds: m and v chain 5 and 6 roundings (the scaled g, 1 - b, the products,
  the sum; nvcc may contract); the step lr_t m / (sqrt v + eps) inherits m's and v's errors plus sqrtf, + eps, the
  quotient, the products and lr_t (rounded once from double); p - step one more; ema - (ema - p)(1 - d) two more."""
  hp = ADAM_HP
  lr, b1, b2, eps, dec = (float(hp[k]) for k in ("lr", "b1", "b2", "eps", "decay"))
  p64, g64, m64, v64, e64 = (d64(a) for a in (p, g, m, v, ema))
  gi = g64 * float(np.float32(ac.gscale))
  m1 = b1 * m64 + (1 - b1) * gi
  v1 = b2 * v64 + (1 - b2) * gi * gi
  em = gamma(5) * (np.abs(b1 * m64) + np.abs((1 - b1) * gi))
  ev = gamma(6) * (np.abs(b2 * v64) + np.abs((1 - b2) * gi * gi))
  lr_t = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
  sq = np.sqrt(v1)
  den = sq + eps
  esq = np.minimum(ev / (2 * np.maximum(sq, 1e-300)), np.sqrt(ev)) + U * sq
  eden = esq + U * den
  step = lr_t * m1 / den
  estep = lr_t * (em / den + np.abs(m1) * eden / den ** 2) + gamma(4) * np.abs(step)
  p1 = p64 - step
  ep = estep + U * np.abs(p1)
  d = dec if ac.ema_on else 0.0
  e1 = e64 - (e64 - p1) * (1 - d)
  ee = (1 - d) * ep + gamma(4) * (np.abs(e64) + np.abs(e64 - p1) * (1 - d))
  return {"p": (p1, ep + TINY), "m": (m1, em + TINY), "v": (v1, ev + TINY), "ema": (e1, ee + TINY)}


def run_adam(K, ac, p, g, m, v, ema, t0, ema_start, lr_t_off=0):
  hp = ADAM_HP
  bufs = {k: Guarded(K, a) for k, a in (("p", p), ("g", g), ("m", m), ("v", v), ("ema", ema))}
  S = Guarded(K, np.array([t0], np.int32).view(np.float32))
  launch(K, 2, "adam_step", bufs["p"].ptr, bufs["g"].ptr, bufs["m"].ptr, bufs["v"].ptr, ac.n, float(hp["lr"]),
         float(hp["b1"]), float(hp["b2"]), float(hp["eps"]), float(np.float32(ac.gscale)), S.ptr, bufs["ema"].ptr,
         float(hp["decay"]), ema_start)
  return bufs, S


def check_adam_case(K, ac):
  """The counter is preset to t - 1 and must read t afterwards; EMA on: ema_start = t - 1 (t - 1 >= ema_start), off:
  ema_start = t.  Each output is judged against one float64 step from the kernel's own fp32 state."""
  p, g, m, v, ema = adam_state(ac)
  t = ac.t
  ref = adam_reference(ac, p, g, m, v, ema, t)
  bufs, S = run_adam(K, ac, p, g, m, v, ema, t - 1, t - 1 if ac.ema_on else t)
  got = S.read()[S.lead:S.lead + 1].view(np.int32)[0]
  assert got == t, "%s: the step counter reads %d after one step from %d" % (ac.id, got, t - 1)
  worst = 0.0
  for k in ("m", "v", "p", "ema"):
    _, r = read(bufs[k], (ac.n,), "%s %s" % (ac.id, k), ("i",), bound=ref[k])
    worst = max(worst, r)
  unchanged(bufs["g"], g, ac.id + " g")
  record(K, "adam_step", ac.id, worst)


# ---------------------------------------------------------------------------------------------------- utilities

def check_utilities(K):
  rng = np.random.RandomState(seed_of("utilities"))
  # fill, copy
  for n in (1, 1001, SWEEP // 4 + 3):
    x = rng.standard_normal(n).astype(np.float32)
    Y = out_buf(K, n)
    launch(K, 1, "fill", Y.ptr, -2.5, n)
    read(Y, (n,), "fill n%d" % n, ("i",), exact=np.full(n, -2.5))
    X, Y = Guarded(K, x), out_buf(K, n)
    launch(K, 1, "copy", Y.ptr, X.ptr, n)
    read(Y, (n,), "copy n%d" % n, ("i",), exact=x)
    record(K, "fill", "n%d" % n)
    record(K, "copy", "n%d" % n)
  # copy2d: column windows of leading dimensions wider than the window; the rest of the destination keeps its bits
  rows, cols, dld, doff, sld, soff = 37, 25, 40, 3, 33, 5
  s = rng.standard_normal((rows, sld)).astype(np.float32)
  d0 = rng.standard_normal((rows, dld)).astype(np.float32)
  S, D = Guarded(K, s), Guarded(K, d0)
  launch(K, 1, "copy2d", D.ptr, dld, doff, S.ptr, sld, soff, rows, cols)
  offs = np.arange(rows)[:, None] * dld + doff + np.arange(cols)[None, :]
  verify(D, offs, s[:, soff:soff + cols], "copy2d", ("row", "col"))
  record(K, "copy2d", "r%d-c%d" % (rows, cols))
  # axpby: y = a x + c (+ b y0): a x + c and b y0 + (...) may each contract into an FMA; three roundings at most
  n = 5003
  x, y0 = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
  a, b, c = np.float32(0.7), np.float32(-1.3), np.float32(0.01)
  for with_y0 in (True, False):
    X, Y0, Y = Guarded(K, x), Guarded(K, y0), out_buf(K, n)
    launch(K, 1, "axpby", Y.ptr, float(a), X.ptr, float(b), Y0.ptr if with_y0 else None, float(c), n)
    y64 = float(a) * d64(x) + float(c) + (float(b) * d64(y0) if with_y0 else 0.0)
    A = abs(float(a)) * np.abs(d64(x)) + abs(float(c)) + (abs(float(b)) * np.abs(d64(y0)) if with_y0 else 0.0)
    _, r = read(Y, (n,), "axpby%s" % (" y0" if with_y0 else ""), ("i",), bound=(y64, gamma(3) * A + TINY))
    record(K, "axpby", "y0" if with_y0 else "no-y0", r)
  # scale_by_dev: x / s per element (inverse, mul 1); else x * f with f = mul / s or mul * s rounded once
  sdev = np.float32(3.0) + np.float32(2.0 ** -20)
  for inverse, mul in ((1, 1.0), (1, 2.5), (0, 1.0), (0, 2.5)):
    X, Sd, Y = Guarded(K, x), Guarded(K, np.array([sdev])), out_buf(K, n)
    launch(K, 1, "scale_by_dev", Y.ptr, X.ptr, Sd.ptr, mul, inverse, n)
    if inverse and mul == 1.0:
      want = (d64(x) / float(sdev)).astype(np.float32)        # correctly rounded quotient (float64 rounds innocuously)
    else:
      f = np.float32(mul) / sdev if inverse else np.float32(mul) * sdev
      want = x * f
    read(Y, (n,), "scale_by_dev inverse %d mul %g" % (inverse, mul), ("i",), exact=want)
    record(K, "scale_by_dev", "inv%d-mul%g" % (inverse, mul))
  # dot: 2 launches; at n = 10^6 the partial grid is capped at 1024 blocks
  for n in (1, 1000, 10 ** 6 + 3):
    a1, b1 = rng.standard_normal(n).astype(np.float32), rng.standard_normal(n).astype(np.float32)
    A1, B1, O = Guarded(K, a1), Guarded(K, b1), out_buf(K, 1)
    launch(K, 2, "dot", O.ptr, A1.ptr, B1.ptr, n)
    blocks = min(-(-n // 256), SMS * 16, 1024)
    L = -(-n // (blocks * 256)) + BLOCK_SUM + -(-blocks // 256) + BLOCK_SUM
    y64 = np.array([(d64(a1) * d64(b1)).sum()])
    _, r = read(O, (1,), "dot n%d" % n, ("i",), bound=(y64, gamma(L) * np.array([(np.abs(d64(a1) * d64(b1))).sum()]) + TINY))
    record(K, "dot", "n%d" % n, r)
  # interpolate: x + alpha (xf - x): the difference, the product (may contract with the sum), the sum
  ns, per = 5, 1001
  x, xf = rng.standard_normal((ns, per)).astype(np.float32), rng.standard_normal((ns, per)).astype(np.float32)
  al = f32([0.0, 1.0, 0.3, 0.999, 0.5])
  X, XF, AL, Y = Guarded(K, x), Guarded(K, xf), Guarded(K, al), out_buf(K, ns * per)
  launch(K, 1, "interpolate", Y.ptr, X.ptr, XF.ptr, AL.ptr, ns, per)
  x64, xf64, a64 = d64(x), d64(xf), d64(al)[:, None]
  y64 = x64 + a64 * (xf64 - x64)
  _, r = read(Y, (ns, per), "interpolate", ("sample", "i"), bound=(y64, gamma(3) * (np.abs(x64) + a64 * (np.abs(xf64) + np.abs(x64))) + TINY))
  record(K, "interpolate", "n%d-per%d" % (ns, per), r)
  # bias_add (c not a power of two), rowscale, one_hot (out-of-range labels give zero rows)
  for c in (3, 33, 100):
    rows = 37
    x, bias = rng.standard_normal((rows, c)).astype(np.float32), rng.standard_normal(c).astype(np.float32)
    X, B, Y = Guarded(K, x), Guarded(K, bias), out_buf(K, rows * c)
    launch(K, 1, "bias_add", Y.ptr, X.ptr, B.ptr, rows, c)
    read(Y, (rows, c), "bias_add c%d" % c, ("row", "c"), exact=x + bias)
    record(K, "bias_add", "c%d" % c)
    s = rng.standard_normal(rows).astype(np.float32)
    Sv, Y = Guarded(K, s), out_buf(K, rows * c)
    launch(K, 1, "rowscale", Y.ptr, X.ptr, Sv.ptr, rows, c)
    read(Y, (rows, c), "rowscale c%d" % c, ("row", "c"), exact=x * s[:, None])
    record(K, "rowscale", "c%d" % c)
  n, classes = 300, 17
  lab = rng.randint(0, classes, n).astype(np.int32)
  lab[:3] = [-1, classes, 0]
  Lb, O = Guarded(K, lab.view(np.float32)), out_buf(K, n * classes)
  launch(K, 1, "one_hot", O.ptr, Lb.ptr, n, classes)
  want = (lab[:, None] == np.arange(classes)[None, :]).astype(np.float32)
  read(O, (n, classes), "one_hot", ("row", "class"), exact=want)
  record(K, "one_hot", "n%d-c%d" % (n, classes))


# ---------------------------------------------------------------------------------------------------- tangents

def check_maxpool2_jvp(K, k):
  """The tangent at the window's first maximum (the cell maxpool2_bwd routes to) of every tangent of the sample."""
  cid = "maxpool2_jvp-k%d" % k
  rng = np.random.RandomState(seed_of(cid))
  n, h, w, c = 3, 6, 8, 5
  x = tie_windows(rng, (n, h, w, c))
  t = rng.standard_normal((n * k, h, w, c)).astype(np.float32)
  X, T, O = Guarded(K, x), Guarded(K, t), out_buf(K, n * k * (h // 2) * (w // 2) * c)
  launch(K, 1, "maxpool2_jvp", O.ptr, T.ptr, X.ptr, n, h, w, c, k)
  arg = np.repeat(first_max(windows(x)), k, axis=0)
  want = np.take_along_axis(windows(t), arg[..., None], -1)[..., 0]
  read(O, want.shape, cid, ("tangent image", "y", "x", "c"), exact=want)
  record(K, "maxpool2_jvp", cid)


def check_act_jvp(K, k):
  """ReLU and leaky ReLU tangents at +-0 (TF's rule, as act_bwd), bit-exact."""
  rng = np.random.RandomState(seed_of("act_jvp", k))
  n, per = 3, 101
  r = rng.standard_normal((n, per)).astype(np.float32)
  r[:, :10:2], r[:, 1:10:2] = 0.0, -0.0
  t = rng.standard_normal((n, k, per)).astype(np.float32)
  for kind in (1, 2):
    R, T, O = Guarded(K, r), Guarded(K, t), out_buf(K, t.size)
    launch(K, 1, "act_jvp", O.ptr, T.ptr, R.ptr, kind, float(LEAK), n, per, k)
    want = relu_gate(np.broadcast_to(r[:, None], t.shape), t, LEAK if kind == 2 else 0.0)
    read(O, t.shape, "act_jvp %s k%d" % (ACT_NAMES[kind], k), ("sample", "tangent", "i"), exact=want)
    record(K, "act_jvp", "%s-k%d" % (ACT_NAMES[kind], k))


SOFTMAX_JVP_CASES = [(2, 3, 77, 4), (3, 2, 256, 2), (1, 4, 1024, 3)]     # (n_primal, rows_per_sample, cols, k)


def check_softmax_jvp(K, n, rps, cols, k):
  """p (t - <t, p>) per tangent row, p of its sample's row: ceil(cols / 256) products per thread, block_sum, the
  difference and the product."""
  cid = "softmax_jvp-n%d-rps%d-c%d-k%d" % (n, rps, cols, k)
  rng = np.random.RandomState(seed_of(cid))
  z = rng.standard_normal((n, rps, cols))
  p = (np.exp(z) / np.exp(z).sum(-1, keepdims=True)).astype(np.float32)
  t = rng.standard_normal((n, k, rps, cols)).astype(np.float32)
  P, T, O = Guarded(K, p), Guarded(K, t), out_buf(K, t.size)
  launch(K, 1, "softmax_jvp", O.ptr, T.ptr, P.ptr, n, rps, cols, k)
  p64, t64 = d64(p)[:, None], d64(t)
  s = (t64 * p64).sum(-1, keepdims=True)
  sa = (np.abs(t64) * p64).sum(-1, keepdims=True)
  L = -(-cols // 256) + BLOCK_SUM + 2
  _, r = read(O, t.shape, cid, ("sample", "tangent", "row", "col"),
              bound=(p64 * (t64 - s), gamma(L) * p64 * (np.abs(t64) + sa) + TINY))
  record(K, "softmax_jvp", cid, r)


# ---------------------------------------------------------------------------------------------------- GPU tests

@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  return kernels


@pytest.mark.gpu
@pytest.mark.parametrize("vc", VEC_CASES, ids=[v.id for v in VEC_CASES])
def test_elementwise_vectors(K, vc):
  (check_act_case if vc.op == "act" else check_add_case)(K, vc)


@pytest.mark.gpu
@pytest.mark.parametrize("pc", POOL_CASES, ids=[p.id for p in POOL_CASES])
def test_pool2(K, pc):
  if pc.vec4:
    check_pool_twin(K, pc)
  else:
    check_pool_case(K, pc)


@pytest.mark.gpu
@pytest.mark.parametrize("pc", POOL2D_CASES, ids=[p.id for p in POOL2D_CASES])
def test_pool2d(K, pc):
  check_pool2d(K, pc)


@pytest.mark.gpu
@pytest.mark.parametrize("n,hw,c,mean", GLOBAL_CASES)
def test_globalpool(K, n, hw, c, mean):
  check_globalpool(K, n, hw, c, mean)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,which,b", LOSS_CASES, ids=[loss_id(*c) for c in LOSS_CASES])
def test_gan_loss(K, kind, which, b):
  check_loss_case(K, kind, which, b)


@pytest.mark.gpu
@pytest.mark.parametrize("n,per", GP_CASES)
def test_gp_penalty(K, n, per):
  check_gp_case(K, n, per)


@pytest.mark.gpu
@pytest.mark.parametrize("rows", ROT_ROWS)
def test_rotation_loss(K, rows):
  check_rotation_case(K, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("rows,wkind", XENT_CASES)
def test_softmax_xent(K, rows, wkind):
  check_xent_case(K, rows, wkind)


@pytest.mark.gpu
def test_s3gan_heads_and_rot90(K):
  check_heads(K)


@pytest.mark.gpu
@pytest.mark.parametrize("ac", ADAM_CASES, ids=[a.id for a in ADAM_CASES])
def test_adam_ema(K, ac):
  check_adam_case(K, ac)


@pytest.mark.gpu
def test_utilities(K):
  check_utilities(K)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3])
def test_tangents(K, k):
  check_maxpool2_jvp(K, k)
  check_act_jvp(K, k)


@pytest.mark.gpu
@pytest.mark.parametrize("n,rps,cols,k", SOFTMAX_JVP_CASES)
def test_softmax_jvp(K, n, rps, cols, k):
  check_softmax_jvp(K, n, rps, cols, k)


# ---------------------------------------------------------------------------------------------------- CPU tests

def test_case_tables_cover_the_edges():
  assert {1, 3, 4, 5} <= {v.n for v in VEC_CASES} and {n % 4 for n in VEC_N if n > 8} == {1, 2, 3}
  assert max(v.n for v in VEC_CASES) > 4 * SMS * 16 * 256
  assert {(v.kind, v.rnd) for v in VEC_CASES if v.op == "act"} == {(k, r) for k in (1, 2, 3, 4) for r in (0, 1)}
  assert any(p.vec4 for p in POOL_CASES) and {1, 3, 5} <= {p.c for p in POOL_CASES}
  assert any(p.mis for p in POOL_CASES) and any(p.h == p.w == 2 for p in POOL_CASES)
  assert any(p.h != p.w for p in POOL_CASES) and any(p.n % 2 for p in POOL_CASES) and any(p.ties for p in POOL_CASES)
  assert {(p.hw, p.stride, p.pad, p.mode) for p in POOL2D_CASES} == {
      (hw, s, pd, m) for hw in (35, 17, 8) for s in (1, 2) for pd in ("SAME", "VALID") for m in (0, 1)}
  assert {1, 9, 36, 64} == {c[1] for c in GLOBAL_CASES}
  assert set(LOSS_B) == {1, 37, 256, 257, 1000, 4096}
  assert {1, 5, 256} == {n for n, _ in GP_CASES} and max(p for _, p in GP_CASES) == 3 * 128 * 128
  assert {4, 255, 256, 257, 1024} == {r for r, _ in XENT_CASES}
  assert {a.t for a in ADAM_CASES} == {1, 2, 3, 1000, 10 ** 6} and any(a.n % 256 for a in ADAM_CASES)
  assert max(a.n for a in ADAM_CASES) > SMS * 16 * 256 and {a.ema_on for a in ADAM_CASES} == {True, False}
  assert {c for _, _, c, _ in SOFTMAX_JVP_CASES} == {77, 256, 1024}
  # the tie windows hold every tie the first-maximum rule has to break
  wv = windows(tie_windows(np.random.RandomState(0), (3, 8, 6, 8))).reshape(-1, 4)
  top = wv == wv.max(1, keepdims=True)
  assert (top.sum(1) == 4).any() and (top.sum(1) == 2).any()
  assert ((wv == 0).all(1) & np.signbit(wv).any(1)).any()
  # the activation inputs hold the leaky tie and TF32 ties
  x = act_operands(2, 64)[0]
  assert (x == 0).sum() >= 2 and np.signbit(x[x == 0]).any()
  assert ((x.view(np.uint32) & 0x1FFF) == 0x1000).sum() >= 6


def test_leaky_relu_gradient_is_tfs():
  """d/dx max(x, leak x) is 1 at x = +-0 (TF's Maximum sends a tie's gradient to x); the old rule, torch's tie split
  0.5 (1 + leak), and the fused dgrad's old leak are both rejected at exactly those elements."""
  vc = Vec("act", 2, 64, 0)
  x, g, ref = act_operands(2, 64)
  want = act_bwd_reference(2, g, ref, LEAK, 0)[0]
  zero = x == 0
  assert same_bits(want[zero], g[zero])
  for old in (np.where(zero, np.float32(0.5) * (np.float32(1) + LEAK) * g, want), np.where(zero, LEAK * g, want)):
    with pytest.raises(AssertionError, match=r"i=0\)"):
      check_bound(old, d64(want), np.zeros(64), vc.id + " old tie rule", ("i",))
  # the oracle's lrelu has the same gradient
  import torch
  from oracle import tf_ops as T
  xt = torch.tensor([0.0, -0.0, 1.0, -1.0], requires_grad=True)
  T.lrelu(xt, 0.2).sum().backward()
  assert xt.grad.tolist() == [1.0, 1.0, 1.0, pytest.approx(0.2)]


def test_criterion_rejects_local_defects():
  """A shifted pool window, the real and fake gradients swapped, a loss mean over b - 1 and Adam's bias correction one
  step off each fail the bounds at a named element."""
  # pools: the window one column to the right
  pc = Pool(2, 8, 8, 4)
  x, g = pool_operands(pc)
  ref = pool_reference(x, g)
  shifted = windows(np.roll(x, -1, axis=2))
  with pytest.raises(AssertionError, match="n=0, y=0, x=0"):
    check_bound(shifted.max(-1), d64(ref["max"]), np.zeros(ref["max"].shape), "shifted max window", ("n", "y", "x", "c"))
  with pytest.raises(AssertionError, match="n=0, y=0, x=0"):
    check_bound(shifted.mean(-1), *ref["avg"], "shifted avg window", ("n", "y", "x", "c"))
  # gan_loss: the accepted float32 evaluation, then its gradient halves swapped and its means taken over b - 1
  b = 4096
  r, f = logits(b, 0), logits(b, 5)
  for kind in (0, 3):
    ref = loss_reference(kind, 0, r, f)
    out4, dl = loss_fp32_model(kind, r, f, b)
    judge_loss("fp32 model", ref, out4, dl)
    with pytest.raises(AssertionError, match=r"half \(0 real, 1 fake\)=0, i=0"):
      judge_loss("swapped", ref, out4, np.concatenate([dl[b:], dl[:b]]))
    with pytest.raises(AssertionError, match="output=0"):
      judge_loss("mean over b - 1", ref, loss_fp32_model(kind, r, f, b - 1)[0], dl)
  # Adam: lr_t with t - 1 in the bias correction
  for t in (2, 1000):
    ac = Adam(1000, t, 0.25, True)
    p, g, m, v, ema = adam_state(ac)
    ref = adam_reference(ac, p, g, m, v, ema, t)
    good = adam_reference(ac, p, g, m, v, ema, t)["p"][0].astype(np.float32)
    check_bound(good, *ref["p"], "Adam", ("i",))
    off = adam_reference(ac, p, g, m, v, ema, t - 1)["p"][0].astype(np.float32)
    with pytest.raises(AssertionError, match="i="):
      check_bound(off, *ref["p"], "Adam bias correction at t - 1", ("i",))


def loss_fp32_model(kind, r, f, mean_b):
  """gan_loss's arithmetic in numpy float32 for the non-saturating and least-squares losses (which = 0), the means taken
  over mean_b."""
  inv = np.float32(1.0) / np.float32(mean_b)
  sig = lambda x: (np.float32(1) / (np.float32(1) + np.exp(-x))).astype(np.float32)
  with np.errstate(over="ignore"):
    pr, pf = sig(r), sig(f)
  if kind == 0:
    sce = lambda x, z: (np.maximum(x, 0) - x * np.float32(z) + np.log1p(np.exp(-np.abs(x)))).astype(np.float32)
    terms = (sce(r, 1), sce(f, 0), sce(f, 1))
    dl = np.concatenate([(pr - 1) * inv, pf * inv])
  else:
    terms = ((pr - 1) ** 2, pf * pf, np.float32(0.5) * (pf - 1) ** 2)
    dl = np.concatenate([(pr - 1) * pr * (1 - pr) * inv, pf * pf * (1 - pf) * inv])
  a, c, gl = (t.sum(dtype=np.float32) * inv for t in terms)
  d = a + c if kind == 0 else np.float32(0.5) * (a + c)
  return f32([d, a, c, gl]), f32(dl)


def test_case_tables_on_the_emulator():
  """Every table through tests/abi_emulator.py: guard bands, layouts, launch bookkeeping and the references agree with
  the C-ABI's contract on the CPU, and the criterion accepts the emulator's arithmetic."""
  from compare_gan_b200 import kernels
  with emulated_library():
    for vc in VEC_CASES:
      if vc.n <= 4096:
        (check_act_case if vc.op == "act" else check_add_case)(kernels, vc)
    for pc in POOL_CASES:
      check_pool_twin(kernels, pc) if pc.vec4 else check_pool_case(kernels, pc)
    for pc in POOL2D_CASES:
      check_pool2d(kernels, pc)
    for c in GLOBAL_CASES:
      check_globalpool(kernels, *c)
    for c in LOSS_CASES:
      check_loss_case(kernels, *c)
    for c in GP_CASES:
      check_gp_case(kernels, *c)
    for rows in ROT_ROWS:
      check_rotation_case(kernels, rows)
    for c in XENT_CASES:
      check_xent_case(kernels, *c)
    check_heads(kernels)
    for ac in ADAM_CASES:
      if ac.n <= 4096:
        check_adam_case(kernels, ac)
    check_utilities(kernels)
    for k in (1, 3):
      check_maxpool2_jvp(kernels, k)
      check_act_jvp(kernels, k)
    for c in SOFTMAX_JVP_CASES:
      check_softmax_jvp(kernels, *c)
