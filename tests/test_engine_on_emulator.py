"""The package's REAL host code — taped ops and their vector-Jacobian products (kernels.py), the tape, flat variable
packing, ModularGAN's unrolled cycle with Adam / EMA / step counters, checkpoints, the schedules of runner_lib — executed
on the CPU against `tests/abi_emulator.py` (a numpy restatement of the C-ABI contract) and compared with the oracle.
No GPU and no CUDA library involved: what is checked here is everything ABOVE the C-ABI; the kernels BELOW it are
checked against the same oracle by the `-m gpu` tests."""
import pytest

from tests.abi_emulator import emulated_library


# The GPU parity tests whose bodies are pure host code + C-ABI calls: the same functions, run against the emulator.
STEP_TESTS = ["test_resnet_cifar_forward", "test_resnet_cifar_cycle_sn_bn", "test_resnet_cifar_cycle_hinge_gsn_ema",
              "test_sndcgan_forward_and_cycle", "test_dcgan_forward_and_cycle", "test_resnet5_wgangp_cycle",
              "test_biggan_forward_and_cycle", "test_biggan_deep_forward_and_cycle",
              "test_initialisation_rules_and_training_determinism"]
EVAL_TESTS = ["test_resize_bilinear_matches_tf_semantics", "test_pool2d_tf_semantics", "test_inception_v3_features",
              "test_train_from_input_pipeline", "test_eval_after_train_schedule_and_checkpoint_roundtrip"]
# math_mode 1 above the emulator (which models the tensor-core ARITHMETIC: TF32-rounded operands, fp32 accumulation):
# the pre-rounding / fused-epilogue plumbing of kernels.py, the in-situ contraction checker and the TF32-emulating oracle
TF32_CASES = ["resnet_cifar", "resnet5_wgangp"]


@pytest.mark.parametrize("name", STEP_TESTS)
def test_training_step_suite_on_the_emulator(name):
  """Forward passes, full cycles (losses, gradients incl. the WGAN-GP double backward, post-Adam weights, EMA, BN state,
  step counters) of every architecture, engine vs oracle — tests/test_gan_step_gpu.py executed above the emulated ABI."""
  import tests.test_gan_step_gpu as gpu_tests
  with emulated_library() as lib:
    getattr(gpu_tests, name)()
    assert lib.launches > 0


@pytest.mark.parametrize("name", EVAL_TESTS)
def test_evaluation_and_schedule_suite_on_the_emulator(name, tmp_path):
  """Resize / pooling semantics, the concat-free Inception-v3 graph, pipeline-fed training, and the eval_after_train
  schedule (training, checkpoint in the reference's key space, FID / IS evaluation of the checkpoint, scores.csv,
  bit-exact checkpoint reload) — tests/test_eval_gpu.py executed above the emulated ABI."""
  import inspect
  import tests.test_eval_gpu as gpu_tests
  from compare_gan_b200 import kernels as K
  fn = getattr(gpu_tests, name)
  with emulated_library():
    fn(K, tmp_path) if "tmp_path" in inspect.signature(fn).parameters else fn(K)


@pytest.mark.parametrize("case", TF32_CASES)
def test_tf32_mode_network_parity_on_the_emulator(case):
  import tests.test_tf32_parity_gpu as gpu_tests
  with emulated_library() as lib:
    gpu_tests.test_tf32_network_parity(case)
    assert lib.launches > 0


def test_inference_mode_generator_and_eval_loop_on_the_emulator():
  """Accumulator fill, EMA weight swap, inference-mode generator and the whole evaluation loop vs oracle/eval.py."""
  import tests.test_eval_gpu as gpu_tests
  from compare_gan_b200 import kernels as K
  with emulated_library():
    gpu_tests.test_inference_mode_generator_and_eval_loop_match_the_oracle(K, "accumulators_and_ema")


def _kernel_test_cases():
  """Every case of tests/test_kernels_gpu.py (parametrisations expanded by hand: the functions are called directly)."""
  import inspect
  import itertools
  import tests.test_kernels_gpu as kt
  for name, fn in inspect.getmembers(kt, inspect.isfunction):
    if not name.startswith("test_"):
      continue
    grids = []
    for mark in [m for m in getattr(fn, "pytestmark", []) if m.name == "parametrize"]:
      names = [n.strip() for n in mark.args[0].split(",")]
      grids.append([dict(zip(names, v if len(names) > 1 else (v,))) for v in mark.args[1]])
    for combo in itertools.product(*grids):
      kw = {}
      for part in combo:
        kw.update(part)
      yield name, fn, kw


def test_emulator_conforms_to_the_kernel_parity_suite():
  """The per-op parity tests define what each C-ABI entry must compute (against the oracle).  Running them against the
  emulator shows that the emulator — on which the host-code tests above rest — honours the same contract.  Only the
  assertions that the tensor-core path was TAKEN (launch counts of the tensor-core kernels) are specific to the real
  library and are skipped."""
  import inspect
  from compare_gan_b200 import kernels as K
  ran = 0
  for name, fn, kw in _kernel_test_cases():
    if "K" in inspect.signature(fn).parameters:
      kw["K"] = K
    try:
      with emulated_library():
        fn(**kw)
    except AssertionError as e:
      msg = str(e)
      path_assertion = ("tcgen05" in name or "tc_" in name) and "rel-L2" not in msg      # "which kernels ran", not numerics
      if not path_assertion:
        raise AssertionError("%s %s: %s" % (name, kw, msg))
    ran += 1
  assert ran > 100


@pytest.mark.parametrize("loss", ["non_saturating", "hinge", "wasserstein", "least_squares"])
def test_every_objective_through_a_full_cycle(loss):
  """modular_gan_test.py:77-80 (testSingleTrainingStepLosses), with numbers: one resnet_cifar cycle per objective, engine
  (loss_lib routing -> fused loss op -> tape) against the oracle."""
  import numpy as np
  from tests.gpu_util import compare_grads, make_inputs, make_pair
  with emulated_library():
    eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 2, d_sn=True, disc_iters=1, loss=loss)
    inputs = make_inputs(np.random.RandomState(11), 1, 2, (32, 32, 3), 128)
    eng.set_inputs(*inputs)
    eng.run_cycle()
    d_losses, g_loss = eng.read_losses()
    ref_d, ref_g = orc.cycle(*inputs)
    assert abs(d_losses[0] - ref_d[0]) <= 1e-4 * max(1.0, abs(ref_d[0])) and abs(g_loss - ref_g) <= 1e-4 * max(1.0, abs(ref_g))
    compare_grads(eng, orc, 2e-3, g_tol=5e-2)


def test_non_unrolled_schedule_matches_the_reference_default():
  """modular_gan.py:534-535, 566-575 (unroll_graph False — the reference's schedule off TPU, modular_gan_test.py:149-177):
  every step is ONE discriminator update on one batch; the generator update runs only when global_step_disc reaches a
  multiple of disc_iters.  Engine (ModularGAN.run_substep) vs oracle (oracle/gan.py substep) over 4 steps at disc_iters
  = 3: losses, which steps updated G, the two step counters, and the state after the last step."""
  import numpy as np
  from tests.gpu_util import compare_states, make_inputs, make_pair
  with emulated_library():
    eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 2, d_sn=True, disc_iters=3, g_use_ema=True, ema_start_step=0)
    rng = np.random.RandomState(5)
    g0 = eng.state_numpy()
    ran_g = []
    for step in range(4):
      imgs, zs, _, _, _ = make_inputs(rng, 3, 2, (32, 32, 3), 128)
      eng.set_inputs(imgs, zs)
      did = eng.run_substep()
      d_losses, g_loss = eng.read_losses()
      ref_d, ref_g = orc.substep(imgs[0], zs[0])
      assert did == (ref_g is not None)
      ran_g.append(did)
      assert abs(d_losses[0] - ref_d) <= 1e-4 * max(1.0, abs(ref_d)), (step, d_losses[0], ref_d)
      if did:
        assert abs(g_loss - ref_g) <= 1e-4 * max(1.0, abs(ref_g)), (step, g_loss, ref_g)
      if step == 1:       # two D updates in, G untouched: its trainable weights are still the initial ones
        s1 = eng.state_numpy()
        assert all(np.array_equal(s1[k], g0[k]) for k in orc.store.trainable if k.startswith("generator/"))
    assert ran_g == [False, False, True, False]
    assert int(eng.d_opt.step.item()) == 4 == orc.global_step_disc and int(eng.g_opt.step.item()) == 1 == orc.global_step
    compare_states(eng, orc, {"generator": 2e-4, "discriminator": 2e-4}, {"generator": 1, "discriminator": 4})


def test_unfed_gradient_penalty_coefficients_come_from_the_library_stream():
  """penalty_lib.wgangp_penalty without a fed `alpha` (reference penalty_lib.py:72-73: tf.random.uniform) draws from
  cgan_random_uniform — no torch RNG on the product path: the penalty of a linear critic equals the closed form evaluated
  with the documented SplitMix64 stream, and a second call continues the stream instead of repeating it."""
  import numpy as np
  from compare_gan_b200 import kernels as K
  from compare_gan_b200.gans import penalty_lib
  with emulated_library():
    rng = np.random.RandomState(0)
    b, d = 6, 12
    x, xf = rng.rand(b, 2, 2, 3).astype(np.float32), rng.rand(b, 2, 2, 3).astype(np.float32)
    w = rng.randn(d, 1).astype(np.float32)
    wd = K.from_numpy(w, req=True)

    def critic(images, y=None, is_training=True, reuse=True):
      logits = K.matmul(K.reshape(images, b, d), wd)
      return K.sigmoid(logits), logits, None
    penalty_lib._ALPHA_RNG["offset"] = 0
    p1 = float(penalty_lib.wgangp_penalty(critic, K.from_numpy(x), K.from_numpy(xf), None, True).cpu()[0])
    assert penalty_lib._ALPHA_RNG["offset"] == b
    p2 = float(penalty_lib.wgangp_penalty(critic, K.from_numpy(x), K.from_numpy(xf), None, True).cpu()[0])
    # a linear critic's input gradient is w for every interpolate: the penalty does not depend on alpha, only its shape does
    want = (np.sqrt(1e-4 + float((w ** 2).sum())) - 1.0) ** 2
    assert abs(p1 - want) <= 1e-5 * max(1.0, want) and abs(p2 - want) <= 1e-5 * max(1.0, want)
    assert penalty_lib._ALPHA_RNG["offset"] == 2 * b
