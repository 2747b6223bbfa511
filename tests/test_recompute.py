"""Recomputed residual / non-local blocks (tape.segment, chosen by ModularGAN.build when the activation stash does not fit):
the segment path must compute what the stash path computes, bit for bit — losses, every parameter, gradient and Adam
moment, the BN moving averages / accumulators, the spectral-norm u vectors, the step counters and the EMA shadow — and its
replays must fire no observer and advance no u vector.  The emulator cases run the package's host code above
tests/abi_emulator.py; the `gpu` cases run the same bodies on the device, eagerly and under CUDA-graph replay, and train
BigGAN-128 at 256 images per GPU.

Run as a script under `torchrun --nproc-per-node 2`, this file is tests/dist_gpu_check.py with segments forced."""
import os
import subprocess
import sys

import numpy as np
import pytest

if __name__ == "__main__":
  sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests.gpu_util import make_inputs, make_pair

_BIGGAN = dict(loss="hinge", g_bn="conditional_batch_norm", g_sn=True, d_sn=True, sn_singular="auto", conditional=True,
               num_classes=10, initializer="orthogonal", use_moving_averages=False, g_lr=1e-4, d_lr=5e-4, beta1=0.0,
               g_use_ema=True, ema_start_step=0, project_y=True)
CASES = {
    # BN in G, SN in D
    "resnet_cifar": dict(arch="resnet_cifar_arch", image=(32, 32, 3), z_dim=128, k=2, pair=dict(d_sn=True)),
    # conditional BN, hierarchical z, attention in G and D, project_y, accumulators, EMA
    "resnet_biggan": dict(arch="resnet_biggan_arch", image=(32, 32, 3), z_dim=120, k=2, classes=10,
                          pair=dict(_BIGGAN, ch=8, extra_bindings=[
                              "resnet_biggan.Generator.blocks_with_attention = 'B2'",
                              "resnet_biggan.Discriminator.blocks_with_attention = 'B1'"])),
    # bottleneck blocks, identity shortcuts, un-chunked z shared by every block, attention at 64x64
    "resnet_biggan_deep": dict(arch="resnet_biggan_deep_arch", image=(64, 64, 3), z_dim=128, k=1, classes=10,
                               pair=dict(_BIGGAN, ch=4)),
    "ssgan": dict(arch="resnet_cifar_arch", image=(32, 32, 3), z_dim=128, k=1, pair=None),
}


def _force(flag):
  """Replaces ModularGAN's memory budget: -1 bytes fits no stash, so build() segments every network it may."""
  from compare_gan_b200.gans import modular_gan
  saved = modular_gan.memory_budget
  if flag:
    modular_gan.memory_budget = lambda: -1
  return saved


def _engine(case, segmented, math_mode=0, batch=2, penalty="no_penalty"):
  from compare_gan_b200.gans import modular_gan
  c = CASES[case]
  saved = _force(segmented)
  try:
    if c["pair"] is None:
      from compare_gan_b200 import datasets, gin_lite as gin
      from compare_gan_b200.gans import ssgan
      gin.clear_config()
      gin.parse_config("\n".join([
          "G.batch_norm_fn = @batch_norm", "D.spectral_norm = True", "standardize_batch.decay = 0.9",
          "standardize_batch.epsilon = 1e-5", "loss.fn = @hinge", "penalty.fn = @%s" % penalty,
          "tf.train.AdamOptimizer.beta1 = 0.5", "ModularGAN.math_mode = %d" % math_mode]))
      ds = datasets.ImageDatasetV2("synthetic", 32, 3, None, 100)
      params = {"architecture": c["arch"], "z_dim": 128, "lambda": 1.0, "disc_iters": c["k"], "seed": 0}
      eng = ssgan.SSGAN(dataset=ds, parameters=params, model_dir="/tmp/cgan_recompute", rotated_batch_size=4 * batch)
      eng.build(batch)
    else:
      eng, _ = make_pair(c["arch"], c["image"], batch, disc_iters=c["k"], z_dim=c["z_dim"], math_mode=math_mode,
                         penalty=penalty, **c["pair"])
  finally:
    modular_gan.memory_budget = saved
  for name in ("generator/non_local_block/sigma", "discriminator/non_local_block/sigma"):
    if name in eng.store.vars:        # open the attention gate so the non-local blocks matter
      eng.store.vars[name].t.fill_(0.5)
  return eng


def _inputs(case, seed, batch=2):
  c = CASES[case]
  return make_inputs(np.random.RandomState(seed), c["k"], batch, c["image"], c["z_dim"], c.get("classes", 0),
                     z_normal="classes" in c)


class _Counting(object):
  """Counts observer calls (RELU_OBSERVERS, ACT_OBSERVERS), segments cut and segment replays."""

  def __init__(self):
    self.relu, self.act, self.cut, self.replays = 0, 0, 0, 0

  def __enter__(self):
    from compare_gan_b200 import kernels as K, tape
    from compare_gan_b200.architectures import arch_ops
    self._K, self._ops, self._tape = K, arch_ops, tape
    self._r = lambda mask: setattr(self, "relu", self.relu + 1)
    self._a = lambda name, y: setattr(self, "act", self.act + 1)
    K.RELU_OBSERVERS.append(self._r)
    arch_ops.ACT_OBSERVERS.append(self._a)
    self._segment, self._replayed = tape.segment, tape.replayed

    def segment(fn, inputs):
      out = self._segment(fn, inputs)
      self.cut += out.node is not None and out.node.name == "segment"
      return out

    def replayed(compute):
      self.replays += tape.replaying()
      return self._replayed(compute)
    tape.segment, tape.replayed = segment, replayed
    K.replayed = replayed
    return self

  def __exit__(self, *a):
    self._K.RELU_OBSERVERS.remove(self._r)
    self._ops.ACT_OBSERVERS.remove(self._a)
    self._tape.segment, self._tape.replayed = self._segment, self._replayed
    self._K.replayed = self._replayed


def _state(eng):
  """Everything a cycle changes, as numpy arrays."""
  s = {"var/" + k: v for k, v in eng.state_numpy().items()}
  for net, flat, opt in (("g", eng.flat_g, eng.g_opt), ("d", eng.flat_d, eng.d_opt)):
    s[net + "/grad"] = flat["grad"].cpu().copy()
    s[net + "/adam_m"], s[net + "/adam_v"] = opt.m.cpu().copy(), opt.v.cpu().copy()
    s[net + "/step"] = opt.step.cpu().numpy().copy()
  if eng.ema is not None:
    s["ema"] = eng.ema.cpu().copy()
  s["losses"] = eng.losses.cpu().copy()
  return s


def _assert_identical(a, b, what):
  assert sorted(a) == sorted(b)
  for k in a:
    np.testing.assert_array_equal(a[k], b[k], err_msg="%s: %s" % (what, k))


def _cycles(eng, case, n=2, counting=None):
  for c in range(n):
    eng.set_inputs(*_inputs(case, 100 + c))
    if counting is None:
      eng.run_cycle()
    else:
      with counting:
        eng.run_cycle()
    eng.read_losses()
  return _state(eng)


def _check_case(case, math_mode=0, graph=False):
  """Two cycles of the stash path and of forced segments on the same seeded inputs: identical state; the segment path cut
  segments in both networks and replayed them, with no observer call and no u_var update beyond the stash path's."""
  from compare_gan_b200 import kernels as K
  try:
    stash = _engine(case, False, math_mode)
    seg = _engine(case, True, math_mode)
    assert stash.recompute == {"generator": False, "discriminator": False}
    assert seg.recompute == {"generator": True, "discriminator": True}
    _assert_identical(_state(stash), _state(seg), "built state")
    if graph:
      stash.capture(warmup=1)
      seg.capture(warmup=1)
      _assert_identical(_cycles(stash, case), _cycles(seg, case), "%s, graph replay, math_mode %d" % (case, math_mode))
      return
    a, b = _Counting(), _Counting()
    s_stash, s_seg = _cycles(stash, case, counting=a), _cycles(seg, case, counting=b)
    _assert_identical(s_stash, s_seg, "%s, math_mode %d" % (case, math_mode))
    assert a.cut == 0 and b.cut > 0 and b.replays > 0, (a.cut, b.cut, b.replays)
    assert (a.relu, a.act) == (b.relu, b.act), "a replay fired observers: %s vs %s" % ((a.relu, a.act), (b.relu, b.act))
  finally:
    K.set_math_mode(0)


def _check_substep(case="resnet_cifar"):
  """The non-unrolled schedule (run_substep) over three steps at disc_iters 2: one of them updates G."""
  stash, seg = _engine(case, False), _engine(case, True)
  ran = []
  for step in range(3):
    for eng in (stash, seg):
      eng.set_inputs(*_inputs(case, 200 + step))
    ran.append((stash.run_substep(), seg.run_substep()))
    _assert_identical(_state(stash), _state(seg), "run_substep %d" % step)
  assert ran == [(False, False), (True, True), (False, False)]


# ---------------------------------------------------------------------------------------------- on the ABI emulator

@pytest.mark.parametrize("case", sorted(CASES))
def test_segments_reproduce_the_stash_path_on_the_emulator(case):
  from tests.abi_emulator import emulated_library
  with emulated_library():
    _check_case(case)


def test_segments_reproduce_the_stash_path_in_tf32_mode_on_the_emulator():
  """math_mode 1: the TF32 pre-rounding decisions (_grad_feeds_tc) and the ReLU-mask fusions across segment borders."""
  from tests.abi_emulator import emulated_library
  with emulated_library():
    _check_case("resnet_biggan", math_mode=1)


def test_non_unrolled_substep_with_segments_on_the_emulator():
  from tests.abi_emulator import emulated_library
  with emulated_library():
    _check_substep()


def test_second_order_penalty_keeps_the_stash_path():
  from tests.abi_emulator import emulated_library
  with emulated_library():
    for penalty in ("wgangp_penalty", "dragan_penalty"):
      assert _engine("resnet_cifar", True, penalty=penalty).recompute == {"generator": False, "discriminator": False}


def test_the_emulator_never_chooses_segments():
  from tests.abi_emulator import emulated_library
  with emulated_library():
    eng = _engine("resnet_biggan", False)
    assert eng.recompute == {"generator": False, "discriminator": False}
    assert not eng.generator.recompute and not eng.discriminator.recompute


def test_segment_is_the_plain_call_outside_a_recorded_network():
  """No segment is cut while the tape does not record, nor in a network that does not recompute."""
  from compare_gan_b200 import tape
  calls = []

  def fn(x):
    calls.append(x)
    return x
  with tape.segments(True), tape.no_record():
    assert tape.segment(fn, ["a"]) == "a"
  with tape.segments(False):
    assert tape.segment(fn, ["b"]) == "b"
  assert calls == ["a", "b"]


# ---------------------------------------------------------------------------------------------- on the GPU

@pytest.mark.gpu
@pytest.mark.parametrize("math_mode", [0, 1])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_segments_reproduce_the_stash_path_gpu(case, graph, math_mode):
  from compare_gan_b200 import kernels as K
  K.init(0)
  _check_case(case, math_mode, graph)


@pytest.mark.gpu
def test_non_unrolled_substep_with_segments_gpu():
  from compare_gan_b200 import kernels as K
  K.init(0)
  _check_substep()


def _biggan256(force):
  """biggan_imagenet128 (ch 96, 128x128, conditional, disc_iters 2, EMA, math_mode 1) built for 256 images per GPU, two
  graph-replayed cycles: (engine, peak device bytes)."""
  import torch
  from compare_gan_b200 import configs, datasets, gin_lite as gin, runner_lib
  from compare_gan_b200.gans import modular_gan
  gin.clear_config()
  gin.parse_config(configs.CONFIGS["biggan_imagenet128"])
  gin.parse_config("ModularGAN.math_mode = 1")
  options = runner_lib.get_options_dict()
  ds = datasets.get_dataset()
  torch.cuda.reset_peak_memory_stats()
  saved = _force(force)
  try:
    eng = options["gan_class"](dataset=ds, parameters=options, model_dir="/tmp/cgan_recompute256").build(256)
  finally:
    modular_gan.memory_budget = saved
  rng = np.random.RandomState(0)
  eng.set_inputs(*runner_lib.sample_cycle_inputs(eng, ds, 256, rng))
  eng.capture(warmup=1)
  for _ in range(2):
    eng.set_inputs(*runner_lib.sample_cycle_inputs(eng, ds, 256, rng))
    eng.run_cycle()
    d_losses, g_loss = eng.read_losses()
    assert np.isfinite(d_losses).all() and np.isfinite(g_loss), (d_losses, g_loss)
  assert eng.global_step == 2 and eng.global_step_disc == 4
  return eng, torch.cuda.max_memory_allocated()


@pytest.mark.gpu
def test_biggan_imagenet128_at_256_images_per_gpu():
  """The reference's 2048 images over 8 GPUs.  build() segments exactly the networks whose predicted stash does not fit
  its budget, and the model trains within the device's memory on the path it chose and with every block recomputed."""
  import gc
  import torch
  from compare_gan_b200 import kernels as K
  K.init(0)
  total = torch.cuda.get_device_properties(0).total_memory
  if total < 70e9:
    pytest.skip("needs an 80 GB device")
  eng, peak = _biggan256(False)
  p = eng.predicted_stash
  fits = lambda g, d: max(p[("discriminator", d)], p[("generator", g)] + p[("discriminator", d)]) <= p["budget"]
  chosen = (eng.recompute["generator"], eng.recompute["discriminator"])
  assert fits(*chosen) or chosen == (True, True), (eng.recompute, p)
  assert chosen == (False, False) or not fits(False, False), (eng.recompute, p)
  assert peak < total
  del eng
  gc.collect()
  torch.cuda.empty_cache()
  seg, seg_peak = _biggan256(True)
  assert seg.recompute == {"generator": True, "discriminator": True}
  assert seg_peak < peak or chosen != (False, False)
  print("biggan_imagenet128 at 256/GPU: chosen %s, peak %.1f GB; every block recomputed: peak %.1f GB (device %.1f GB)"
        % (chosen, peak / 1e9, seg_peak / 1e9, total / 1e9))


@pytest.mark.gpu
def test_data_parallel_equivalence_with_segments_forced():
  import torch
  if torch.cuda.device_count() < 2:
    pytest.skip("needs two GPUs")
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-port", "29533",
                      os.path.abspath(__file__)], cwd=root, capture_output=True, text=True, timeout=900)
  assert r.returncode == 0 and "DIST_EQUIVALENCE PASS" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


if __name__ == "__main__":
  from compare_gan_b200.gans import modular_gan
  from tests import dist_gpu_check
  modular_gan.memory_budget = lambda: -1
  dist_gpu_check.main()
