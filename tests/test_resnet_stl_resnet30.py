"""The resnet_stl (48x48) and resnet30 (128x128, 30 blocks) architectures, and the filter gradients over pixel grids
whose width 32 does not divide that resnet_stl needs on the tensor cores.

CPU: parameter counts at the reference's width, the variable key space against the oracle restatement
(tests/resnet_stl_resnet30_oracle.py), the kernel-call traces pinned in tests/golden/resnet_stl_resnet30.json, and the
engine against the oracle above the emulated C-ABI (forward passes and full cycles, one with D.layer_norm under WGAN-GP).
GPU: every new filter-gradient geometry element by element against float64, both networks against the oracle in
math_mode 0 and resnet_stl in math_mode 1 (see TF32_CASES), plus CUDA-graph replay."""
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import nets as onets
from tests import arch_trace as at
from tests import layer_norm_oracle as lno
from tests import resnet_stl_resnet30_oracle  # noqa: F401  (adds the two pairs to the oracle's tables)
from tests.abi_emulator import emulated_library
from tests.gpu_util import make_inputs, make_pair

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_PATH = os.path.join(HERE, "golden", "resnet_stl_resnet30.json")

STL, R30 = "resnet_stl_arch", "resnet30_arch"


def _ch_bindings(module, ch):
  return ["%s.Generator.ch = %d" % (module, ch), "%s.Discriminator.ch = %d" % (module, ch)]


# ------------------------------------------------------------------------------------------ definitions (CPU)

def _counts(variables):
  g = sum(int(np.prod(s)) for n, s, t in variables if t and n.startswith("generator/"))
  d = sum(int(np.prod(s)) for n, s, t in variables if t and n.startswith("discriminator/"))
  return g, d


def _oracle_variables(arch, image_shape, ch, g_bn=None, z_dim=128):
  cfg = onets.Cfg(architecture=arch, image_shape=image_shape, g_bn=g_bn, ch=ch)
  store = onets.VarStore()
  with torch.no_grad():
    img = onets.generator(store, cfg, torch.zeros(1, z_dim), None, True)
    onets.discriminator(store, cfg, img, None, True)
  return [[k, list(v.shape), k in store.trainable] for k, v in store.vars.items()]


# resnet_stl.py / resnet30.py at ch = 64, z_dim 128, no batch norm: trainable weights of G and D
PARAMETER_COUNTS = [(STL, (48, 48, 3), 6251523, 25114817), (STL, (48, 48, 1), 6250369, 25112513),
                    (R30, (128, 128, 3), 52176531, 53486449), (R30, (128, 128, 1), 52176241, 53486161)]


@pytest.mark.parametrize("arch,image_shape,g,d", PARAMETER_COUNTS)
def test_parameter_counts_at_the_reference_width(arch, image_shape, g, d):
  tr = at.trace_networks("G.batch_norm_fn = None", arch, image_shape)
  engine = [v[:3] for v in tr["variables"]]
  assert _counts(engine) == (g, d)
  assert engine == _oracle_variables(arch, image_shape, 64), "engine and oracle key spaces differ"


# the configurations whose traces are pinned: batch norm in G, spectral norm in D, small widths where the structure
# allows (the trace is shape-only, but initial values are really drawn)
TRACE_CASES = {
    "resnet_stl": dict(gin_text="G.batch_norm_fn = @batch_norm\nD.spectral_norm = True\nresnet_stl.Generator.ch = 16\n"
                                "resnet_stl.Discriminator.ch = 16", architecture=STL, image_shape=(48, 48, 3)),
    "resnet_stl_gray": dict(gin_text="G.batch_norm_fn = @batch_norm\nresnet_stl.Generator.ch = 16\n"
                                     "resnet_stl.Discriminator.ch = 16", architecture=STL, image_shape=(48, 48, 1)),
    "resnet30": dict(gin_text="G.batch_norm_fn = @batch_norm\nD.spectral_norm = True\nresnet30.Generator.ch = 16\n"
                              "resnet30.Discriminator.ch = 16", architecture=R30, image_shape=(128, 128, 3)),
    "resnet30_cbn": dict(gin_text="G.batch_norm_fn = @conditional_batch_norm\nG.spectral_norm = True\n"
                                  "resnet30.Generator.ch = 8\nresnet30.Discriminator.ch = 8", architecture=R30,
                         image_shape=(128, 128, 3), num_classes=10, conditional=True),
}


def write_golden(path=GOLDEN_PATH):
  """Regenerates the golden traces from the CURRENT definitions (only after an intended change)."""
  golden = {"_about": "Traces of the resnet_stl / resnet30 definitions recorded by tests/arch_trace.py; see "
                      "tests/test_resnet_stl_resnet30.py:TRACE_CASES."}
  for name, kw in TRACE_CASES.items():
    tr = at.trace_networks(**kw)
    golden[name] = {"variables": tr["variables"], "n_ops": len(tr["ops"]), "ops_sha1": at.canonical_sha1(tr["ops"])}
  json.dump(golden, open(path, "w"), indent=0)


@pytest.mark.parametrize("case", sorted(TRACE_CASES))
def test_definition_trace_is_pinned(case):
  want = json.load(open(GOLDEN_PATH))[case]
  tr = at.trace_networks(**TRACE_CASES[case])
  assert [v[:3] for v in tr["variables"]] == [v[:3] for v in want["variables"]], "variable names / shapes / trainability"
  assert tr["variables"] == want["variables"], "initial values (initialiser kind or RNG order changed)"
  assert len(tr["ops"]) == want["n_ops"]
  assert at.canonical_sha1(tr["ops"]) == want["ops_sha1"], "kernel-call sequence changed"


def test_block_names_and_shapes_match_the_oracle_with_batch_norm():
  for arch, shape in ((STL, (48, 48, 3)), (R30, (128, 128, 3))):
    module = arch[:-len("_arch")]
    tr = at.trace_networks("G.batch_norm_fn = @batch_norm\n" + "\n".join(_ch_bindings(module, 8)), arch, shape)
    assert [v[:3] for v in tr["variables"]] == _oracle_variables(arch, shape, 8, g_bn="batch_norm")
  names = [v[0] for v in tr["variables"]]
  assert "generator/B_0_4/bn1/gamma" in names and "generator/B_4_up/up_conv1/kernel" in names
  assert "discriminator/color_conv/kernel" in names and "discriminator/B_4_up/down_conv2/kernel" in names
  assert "generator/final_norm/gamma" not in names


def test_input_side_checks():
  from compare_gan_b200.architectures import resnet30, resnet_stl
  from compare_gan_b200 import gin_lite as gin
  gin.clear_config()
  with at.traced_kernels():
    from compare_gan_b200 import variables as V
    with V.use(V.VariableStore(seed=0)):
      with pytest.raises(ValueError, match="power of 2"):
        resnet30.Discriminator(ch=8)(at.FakeDT((2, 48, 48, 3)), None, True)
      _, _, feat = resnet_stl.Discriminator(ch=8)(at.FakeDT((2, 48, 48, 3)), None, True)
      assert feat.shape == (2, 128)
      with pytest.raises(ValueError, match="equal width and height"):
        resnet_stl.Discriminator(ch=8, name="d2")(at.FakeDT((2, 48, 40, 3)), None, True)
      with pytest.raises(ValueError, match="color channels"):
        resnet_stl.Discriminator(ch=8, name="d3")(at.FakeDT((2, 48, 48, 2)), None, True)


# ------------------------------------------------------------------------------------------ networks vs the oracle

_WGANGP = dict(loss="wasserstein", penalty="wgangp_penalty", lamba=10.0, g_lr=1e-4, beta1=0.5, beta2=0.9)


def _stl(colors=3, batch=4, ch=8, extra=(), **kw):
  from tests.test_gan_step_gpu import _cycles_both, _forward_both
  shape = (48, 48, colors)
  # one D step per cycle: the D gradients compared are taken at identical weights (the 1-channel B0 layer's gradients
  # are small enough that a D step earlier in the cycle moves them by more than the tight bound)
  eng, orc = make_pair(STL, shape, batch, disc_iters=1, ch=ch, extra_bindings=_ch_bindings("resnet_stl", ch) + list(extra),
                       **kw)
  _forward_both(eng, orc, batch, 128)
  gp = kw.get("penalty") == "wgangp_penalty"
  _cycles_both(eng, orc, batch, shape, 128, 1, gp=gp, g_lr=kw.get("g_lr", 2e-4), grad_tol=2e-3 if gp else 1e-3,
               loss_tol=3e-3 if gp else 1e-3)


def _r30(batch=2, ch=8, **kw):
  """Thirty residual blocks without a final norm: the fp32 oracle's own G gradients sit far from float64 (worst tensor
  ~0.8 rel-L2 at ch = 8), so the cycle is checked with D frozen against the float64 oracle, calibrated by what the fp32
  oracle loses, rather than fp32 against fp32 after diverging D updates."""
  from tests.test_gan_step_gpu import _forward_both, _frozen_d_gradients
  shape = (128, 128, 3)
  bindings = _ch_bindings("resnet30", ch)
  eng, orc = make_pair(R30, shape, batch, disc_iters=1, ch=ch, extra_bindings=bindings, **kw)
  _forward_both(eng, orc, batch, 128)
  _frozen_d_gradients(batch, shape, 128, 1, arch=R30, ch=ch, extra_bindings=bindings, **kw)


def _stl_layer_norm_wgangp(ch=8):
  with lno.discriminator_layer_norm():
    _stl(ch=ch, extra=[lno.BINDING], **_WGANGP)


NETWORK_CASES = {
    "resnet_stl_rgb_sn": lambda: _stl(3, d_sn=True),
    "resnet_stl_gray": lambda: _stl(1),
    "resnet_stl_layer_norm_wgangp": _stl_layer_norm_wgangp,
    "resnet30_rgb_sn": lambda: _r30(d_sn=True),
}


@pytest.fixture
def emulated_with_layer_norm(monkeypatch):
  from tests.test_layer_norm import _patch
  _patch(monkeypatch.setattr)
  with emulated_library() as lib:
    yield lib


@pytest.mark.parametrize("case", sorted(NETWORK_CASES))
def test_networks_match_the_oracle_on_the_emulator(emulated_with_layer_norm, case):
  NETWORK_CASES[case]()
  assert emulated_with_layer_norm.launches > 0


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(NETWORK_CASES))
def test_networks_match_the_oracle(case):
  NETWORK_CASES[case]()


# math_mode 1 at a width where the 48-pixel grids reach the wgmma filter-gradient kernel (cin >= 64).  resnet30 is not
# among them: its generator's activations pass the check's relative criterion (within 2x of what the TF32-emulating
# oracle loses) but exceed its absolute depth-scaled cap, 4e-4 sqrt(depth + 1), already five blocks in (1.58e-3 against
# 1.55e-3 at generator/B_0_4/same_conv1, ch 16); that cap was set for networks a sixth as deep.
TF32_CASES = {
    "resnet_stl": dict(arch=STL, image=(48, 48, 3), batch=4, z_dim=128, k=1,
                       pair=dict(d_sn=True, ch=32, extra_bindings=_ch_bindings("resnet_stl", 32))),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(TF32_CASES))
def test_tf32_networks_match_the_oracle(monkeypatch, case):
  """The CONV_TRACE-informed check of tests/test_tf32_parity_gpu.py: forward activations against a TF32-emulating
  oracle, every contraction of a cycle recomputed in situ, gradients against float64."""
  import tests.test_tf32_parity_gpu as tf32_tests
  monkeypatch.setitem(tf32_tests.ARCHS, case, TF32_CASES[case])
  tf32_tests.test_tf32_network_parity(case)


@pytest.mark.gpu
@pytest.mark.parametrize("arch,shape,ch,math_mode", [(STL, (48, 48, 3), 32, 1), (R30, (128, 128, 3), 8, 0)])
def test_cuda_graph_replay_equals_eager(arch, shape, ch, math_mode):
  from compare_gan_b200 import kernels as K
  module = arch[:-len("_arch")]
  eng, _ = make_pair(arch, shape, 4, d_sn=True, disc_iters=2, ch=ch, extra_bindings=_ch_bindings(module, ch),
                     math_mode=math_mode)
  try:
    rng = np.random.RandomState(9)
    batches = [make_inputs(rng, 2, 4, shape, 128) for _ in range(2)]
    snap = eng.snapshot()
    eager = []
    for b in batches:
      eng.set_inputs(*b)
      eng.run_cycle()
      eager.append(eng.read_losses())
    state_eager = eng.state_numpy()
    eng.restore(snap)
    eng.capture(warmup=2)
    n0 = K.lib().launch_count()
    for i, b in enumerate(batches):
      eng.set_inputs(*b)
      eng.run_cycle()
      assert eng.read_losses() == eager[i], "graph replay must be bit-identical to eager"
    assert K.lib().launch_count() == n0, "replay launches no new host-side kernels"
    for k, v in eng.state_numpy().items():
      np.testing.assert_array_equal(v, state_eager[k], err_msg=k)
  finally:
    K.set_math_mode(0)


# ------------------------------------------------------------------------------------------ filter-gradient geometry

def _box(n, h, w):
  """The k-block box csrc/wgrad_tc.cu takes for an n x h x w grid (box32, else box_any)."""
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


def _pick_bn(ncols):
  if ncols <= 256 and ncols % 4 == 0:
    return -(-ncols // 32) * 32
  return 256 if ncols % 256 == 0 else 192 if ncols % 192 == 0 else 128


def _wgrad_kernel_launches(n, gh, gw, xch, dych, ntaps, same_b, sms):
  """Launches of one cgan_wgrad_tc call: the kernel, plus the split-K reduction when the pixel range is split."""
  bw, bh, bni = _box(n, gh, gw)
  kblocks = -(-gw // bw) * -(-gh // bh) * -(-n // bni)
  bn = _pick_bn(dych)
  units = -(-xch // 128) * ntaps
  mt = 2 if same_b and units >= 2 and 2 * bn <= 256 else 1
  tiles = -(-dych // bn) * -(-units // mt)
  splits = max(1, min((2 * sms) // tiles, max(kblocks // 8, 1)))
  per = -(-kblocks // splits)
  return 1 + (-(-kblocks // per) > 1)


def test_box_rule_keeps_power_of_two_grids_and_fills_the_48_pixel_pyramid():
  assert _box(2, 16, 8) == (8, 4, 1) and _box(32, 16, 16) == (16, 2, 1)
  for side, box in ((48, (16, 2, 1)), (24, (8, 4, 1)), (12, (4, 4, 2)), (6, (2, 2, 8)), (3, (1, 1, 32))):
    assert _box(64, side, side) == box
    assert math.prod(box) == 32 and side % box[0] == 0 and side % box[1] == 0     # every MMA row a real pixel


def _geometry_cases():
  from tests.test_tc_exact_gpu import wgrad
  return [
      # 3x3 stride-1 convolutions over the resnet_stl maps (at 6x6 batch 1 the box hangs over the bottom row, at 3x3
      # batch 4 over the batch; at 3x3 batch 64 every k-block is 32 images of one pixel)
      wgrad("wgrad", 2, 48, 48, 64, 64, 3, 3),
      wgrad("wgrad", 4, 24, 24, 128, 128, 3, 3),
      wgrad("wgrad", 4, 12, 12, 256, 256, 3, 3),
      wgrad("wgrad", 4, 6, 6, 512, 512, 3, 3),
      wgrad("wgrad", 1, 6, 6, 64, 96, 3, 3),
      wgrad("wgrad", 4, 3, 3, 512, 1024, 3, 3),
      wgrad("wgrad", 64, 3, 3, 128, 64, 3, 3),
      # up-sampling convolutions: the dY phase grids of 6 -> 12, 12 -> 24 and 24 -> 48
      wgrad("wgrad up", 4, 6, 6, 512, 256, 3, 3, up=True),
      wgrad("wgrad up", 4, 12, 12, 256, 128, 3, 3, up=True),
      wgrad("wgrad up", 2, 24, 24, 128, 64, 3, 3, up=True),
      # the image-side layers at 48
      wgrad("wgrad thin-cin", 2, 48, 48, 3, 64, 3, 3),
      wgrad("wgrad thin-cin", 2, 48, 48, 1, 64, 3, 3),
      wgrad("wgrad thin-cout", 2, 48, 48, 64, 3, 3, 3),
      wgrad("wgrad thin-cout", 2, 48, 48, 64, 1, 3, 3),
  ]


def _expected_launches(c, sms):
  if c.path == "wgrad thin-cin":       # patch gather, GEMM over the 32-wide patch rows, copy of the HWIO rows
    return 2 + _wgrad_kernel_launches(c.n, c.h, c.w, 32, c.cout, 1, True, sms)
  if c.path == "wgrad thin-cout":      # patch gather of dY, GEMM, re-layout to HWIO
    return 2 + _wgrad_kernel_launches(c.n, c.h, c.w, c.cin, 32, 1, True, sms)
  return _wgrad_kernel_launches(c.n, c.h, c.w, c.cin, c.cout, c.kh * c.kw, not c.up, sms)


GEOMETRY_IDS = [c.id for c in _geometry_cases()]


@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  kernels.set_math_mode(1)
  yield kernels
  kernels.set_math_mode(0)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(GEOMETRY_IDS)), ids=GEOMETRY_IDS)
def test_wgrad_over_grids_32_does_not_divide_elementwise(K, i):
  from tests import test_tc_exact_gpu as tce
  c = _geometry_cases()[i]
  c.launches = _expected_launches(c, torch.cuda.get_device_properties(0).multi_processor_count)
  tce.check_case(K, c)
