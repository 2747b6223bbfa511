"""Shared helpers for the -m gpu parity tests: build the engine (CUDA, through the C-ABI) and the CPU oracle
with identical configuration and identical initial weights."""
import numpy as np
import torch

from oracle import gan as ogan
from oracle import nets as onets


def rel_err(a, b):
  a = np.asarray(a, np.float64)
  b = np.asarray(b, np.float64)
  d = np.linalg.norm((a - b).ravel())
  n = np.linalg.norm(b.ravel())
  return d / max(n, 1e-30)


def assert_close(a, b, tol, what=""):
  a, b = np.asarray(a), np.asarray(b)
  assert a.shape == b.shape, "%s: shape %s vs %s" % (what, a.shape, b.shape)
  e = rel_err(a, b)
  assert np.isfinite(a).all(), "%s: non-finite values" % what
  assert e <= tol, "%s: rel-L2 error %.3e > %.1e" % (what, e, tol)


ARCH_IMAGE = {"resnet_cifar_arch": (32, 32, 3)}


def make_pair(arch, image_shape, batch, loss="non_saturating", penalty="no_penalty", lamba=1.0, disc_iters=1,
              g_bn="batch_norm", g_sn=False, d_sn=False, sn_singular="left", conditional=False, num_classes=0,
              initializer="normal", use_moving_averages=True, bn_decay=0.9, bn_eps=1e-5, g_lr=2e-4, d_lr=None,
              beta1=0.5, beta2=0.999, z_dim=128, g_use_ema=False, ema_start_step=0, ch=8, extra_bindings=(),
              project_y=False, seed=0, with64=False, math_mode=0):
  """Returns (engine ModularGAN built for `batch`, GanOracle) sharing config and weights."""
  from compare_gan_b200 import gin_lite as gin
  from compare_gan_b200 import datasets
  from compare_gan_b200.gans import modular_gan  # noqa: F401  (registers configurables)
  gin.clear_config()
  bn_ref = {"batch_norm": "@batch_norm", "conditional_batch_norm": "@conditional_batch_norm", None: "None"}[g_bn]
  cfg = [
      "G.batch_norm_fn = %s" % bn_ref,
      "G.spectral_norm = %s" % g_sn,
      "D.spectral_norm = %s" % d_sn,
      "spectral_norm.singular_value = '%s'" % sn_singular,
      "standardize_batch.decay = %r" % bn_decay,
      "standardize_batch.epsilon = %r" % bn_eps,
      "standardize_batch.use_moving_averages = %s" % use_moving_averages,
      "weights.initializer = '%s'" % initializer,
      "loss.fn = @%s" % loss,
      "penalty.fn = @%s" % penalty,
      "ModularGAN.g_lr = %r" % g_lr,
      "ModularGAN.g_optimizer_fn = @tf.train.AdamOptimizer",
      "tf.train.AdamOptimizer.beta1 = %r" % beta1,
      "tf.train.AdamOptimizer.beta2 = %r" % beta2,
      "ModularGAN.conditional = %s" % conditional,
      "ModularGAN.g_use_ema = %s" % g_use_ema,
      "ModularGAN.ema_start_step = %d" % ema_start_step,
      "resnet_biggan.Generator.ch = %d" % ch,
      "resnet_biggan.Discriminator.ch = %d" % ch,
      "resnet_biggan.Discriminator.project_y = %s" % project_y,
      "resnet_biggan_deep.Generator.ch = %d" % ch,
      "resnet_biggan_deep.Discriminator.ch = %d" % ch,
      "resnet_biggan_deep.Discriminator.project_y = %s" % project_y,
      "resnet_cifar.Discriminator.project_y = %s" % project_y,
      "ModularGAN.math_mode = %d" % math_mode,
  ]
  if d_lr is not None:
    cfg.append("ModularGAN.d_lr = %r" % d_lr)
  cfg += list(extra_bindings)
  gin.parse_config("\n".join(cfg))
  ds = datasets.ImageDatasetV2("synthetic", image_shape[0], image_shape[2], num_classes or None, 100)
  params = {"architecture": arch, "z_dim": z_dim, "lambda": lamba, "disc_iters": disc_iters, "seed": seed}
  eng = modular_gan.ModularGAN(dataset=ds, parameters=params, model_dir="/tmp/cgan_test")
  eng.build(batch)

  hier = arch == "resnet_biggan_arch"
  ocfg = onets.Cfg(architecture=arch, image_shape=tuple(image_shape), g_bn=g_bn, g_sn=g_sn, d_sn=d_sn,
                   sn_singular=sn_singular, bn_decay=bn_decay, bn_eps=bn_eps,
                   use_moving_averages=use_moving_averages, initializer=initializer, ch=ch, project_y=project_y,
                   hierarchical_z=hier, embed_y=hier or arch == "resnet_biggan_deep_arch", num_classes=num_classes)
  for b in extra_bindings:
    if "Generator.blocks_with_attention" in b:
      ocfg.g_attention = b.split("=")[1].strip().strip("'\"")
    if "Discriminator.blocks_with_attention" in b:
      ocfg.d_attention = b.split("=")[1].strip().strip("'\"")
  orc = ogan.GanOracle(ocfg, loss=loss, penalty=penalty, lamba=lamba, disc_iters=disc_iters, g_lr=g_lr, d_lr=d_lr,
                       beta1=beta1, beta2=beta2, conditional=conditional, g_use_ema=g_use_ema,
                       ema_start_step=ema_start_step, z_dim=z_dim).build(batch)
  state = eng.state_numpy()
  onames = list(orc.store.vars.keys())
  enames = list(state.keys())
  assert sorted(onames) == sorted(enames), ("variable sets differ", sorted(set(onames) ^ set(enames))[:10])
  assert [k for k in orc.store.trainable] == [k for k in eng.store.trainable], "trainable variable order differs"
  orc.store.load_numpy(state)
  if with64:   # float64 twin of the oracle: the yard-stick for what fp32 rounding alone does to a gradient
    orc64 = ogan.GanOracle(ocfg, loss=loss, penalty=penalty, lamba=lamba, disc_iters=disc_iters, g_lr=g_lr, d_lr=d_lr,
                           beta1=beta1, beta2=beta2, conditional=conditional, g_use_ema=g_use_ema,
                           ema_start_step=ema_start_step, z_dim=z_dim, dtype=torch.float64).build(batch)
    orc64.store.load_numpy(state)
    return eng, orc, orc64
  return eng, orc


def make_inputs(rng, k, batch, image_shape, z_dim, num_classes=0, z_normal=False, gp=False):
  imgs = [rng.rand(batch, *image_shape).astype(np.float32) for _ in range(k + 1)]
  if z_normal:
    zs = [rng.standard_normal((batch, z_dim)).astype(np.float32) for _ in range(k + 1)]
  else:
    zs = [rng.uniform(-1, 1, (batch, z_dim)).astype(np.float32) for _ in range(k + 1)]
  labels = sampled = None
  if num_classes:
    labels = [rng.randint(0, num_classes, batch).astype(np.int32) for _ in range(k + 1)]
    sampled = [rng.randint(0, num_classes, batch).astype(np.int32) for _ in range(k + 1)]
  alphas = [rng.rand(batch, 1, 1, 1).astype(np.float32) for _ in range(k + 1)] if gp else None
  return imgs, zs, labels, sampled, alphas


class ReluSigns(object):
  """Records the sign pattern of every ReLU / leaky-ReLU input, on the engine (K.act) and on the oracle
  (torch.relu / tf_ops.lrelu).  A ReLU input that sits within rounding distance of zero takes a different branch in
  two correct fp32 implementations, and that single mask flip changes the gradients discontinuously (measured: one
  flipped element out of 262144 moves a generator gradient by 5e-3 rel-L2).  Gradient parity is therefore asserted
  at the tight tolerance only when the masks agree, and at a loose one otherwise."""

  def __init__(self):
    self.eng, self.orc = [], []

  def __enter__(self):
    from compare_gan_b200 import kernels as K
    from oracle import tf_ops as T
    self._K, self._T = K, T
    self._relu, self._lrelu = torch.relu, T.lrelu
    rec = self
    self._obs = lambda mask: rec.eng.append(mask.cpu().numpy())
    K.RELU_OBSERVERS.append(self._obs)

    def relu(x):
      rec.orc.append((x.detach() > 0).numpy())
      return rec._relu(x)

    def lrelu(x, leak=0.2):
      rec.orc.append((x.detach() > 0).numpy())
      return rec._lrelu(x, leak)
    torch.relu, T.lrelu = relu, lrelu
    return self

  def __exit__(self, *a):
    self._K.RELU_OBSERVERS.remove(self._obs)
    torch.relu, self._T.lrelu = self._relu, self._lrelu

  def start_oracle(self):
    self.orc = []

  def flips(self):
    assert len(self.eng) == len(self.orc), (len(self.eng), len(self.orc))
    return int(sum(int((a != b).sum()) for a, b in zip(self.eng, self.orc)))


def compare_grads(eng, orc, tol=1e-3, g_tol=None, orc64=None, flips=0):
  """Gradients of the last D-update and of the G-update (flat buffers) vs the oracle's autograd gradients.
  Per tensor: ||g - g_ref|| <= tol * ||g_ref|| + 1e-5 * (largest tensor-gradient norm of that network); the absolute
  floor covers parameters whose true gradient is zero (e.g. a conv bias that feeds a BatchNorm), where both sides
  hold only rounding noise."""
  worst = (0.0, None)
  if flips:
    tol = max(tol, 5e-2)       # ReLU masks differ in `flips` elements: only a loose bound is meaningful
  for prefix, flat, ref in (("discriminator", eng.flat_d, orc.last_d_grads), ("generator", eng.flat_g, orc.last_g_grads)):
    if orc64 is not None:
      # against the float64 gradients, allowing what the fp32 CPU oracle itself loses to rounding (x4)
      ref64 = orc64.last_d_grads if prefix == "discriminator" else orc64.last_g_grads
      g = flat["grad"].cpu()
      gmax = max(float(v.norm()) for v in ref64.values())
      for name, (off, n) in flat["views"].items():
        a, b64, b32 = g[off:off + n].astype(np.float64), ref64[name].numpy().ravel(), ref[name].numpy().ravel().astype(np.float64)
        assert np.isfinite(a).all(), name
        err, err32 = np.linalg.norm(a - b64), np.linalg.norm(b32 - b64)
        bound = tol * np.linalg.norm(b64) + 1e-5 * gmax + 4.0 * err32
        assert err <= bound, "%s grad vs fp64: |err| %.3e > %.3e (|ref| %.3e, fp32-oracle err %.3e)" % (
            name, err, bound, np.linalg.norm(b64), err32)
        if np.linalg.norm(b64) > 1e-3 * gmax:
          worst = max(worst, (err / np.linalg.norm(b64), name))
      continue
    g = flat["grad"].cpu()
    gmax = max(float(v.norm()) for v in ref.values())
    for name, (off, n) in flat["views"].items():
      a, b = g[off:off + n], ref[name].numpy().ravel()
      assert np.isfinite(a).all(), name
      err = np.linalg.norm(a.astype(np.float64) - b)
      bound = (tol if prefix == "discriminator" or g_tol is None else g_tol) * np.linalg.norm(b) + 1e-5 * gmax
      assert err <= bound, "%s grad: |err| %.3e > %.3e (|ref| %.3e, net max %.3e)" % (name, err, bound, np.linalg.norm(b), gmax)
      if np.linalg.norm(b) > 1e-3 * gmax:
        worst = max(worst, (err / np.linalg.norm(b), name))
  return worst


def compare_states(eng, orc, lr, updates, frac=0.35, skip=(), state_tol=2e-3):
  """Weights after Adam.  Adam's first steps move every element by ~lr*sign(g): elements whose gradient is at the
  rounding-noise level flip sign in ANY two implementations, so the criterion is in units of the step size:
  rms(w - w_ref) <= frac * lr * updates per tensor; tensors whose reference gradient is pure noise are skipped."""
  es = eng.state_numpy()
  refg = {}
  refg.update(getattr(orc, "last_d_grads", {}) or {})
  refg.update(getattr(orc, "last_g_grads", {}) or {})
  gmax = {"generator": 1e-30, "discriminator": 1e-30}
  for k, v in refg.items():
    gmax[k.split("/")[0]] = max(gmax[k.split("/")[0]], float(v.norm()))
  worst = (0.0, None)
  for k, v in orc.store.vars.items():
    if any(s in k for s in skip):
      continue
    a, b = es[k], v.detach().numpy()
    assert np.isfinite(a).all(), k
    if k in orc.store.trainable:
      if k in refg and float(refg[k].norm()) < 1e-4 * gmax[k.split("/")[0]]:
        continue   # noise-dominated gradient (zero in exact arithmetic)
      rms = float(np.sqrt(np.mean((a.astype(np.float64) - b) ** 2)))
      lim = frac * lr[k.split("/")[0]] * updates[k.split("/")[0]]
      if rms / lim >= worst[0]:
        worst = (rms / lim, k)
      assert rms <= lim, "%s: rms weight error %.3e > %.3e" % (k, rms, lim)
    else:
      e = rel_err(a, b)
      assert e <= state_tol, "%s (state): rel-L2 error %.3e" % (k, e)
  return worst
