"""Gradient penalties (reference gans/penalty_lib.py:28-108)."""
from .. import gin_lite as gin
from .. import kernels as K
from .. import tape
from .. import utils


_ALPHA_RNG = {"seed": 0x5EEDA1FA, "offset": 0}     # stream of the un-fed interpolation coefficients (per process)
# stream of DRAGAN's perturbation (plus the replica id); its offset is the discriminator's step counter times numel(x)
DRAGAN_SEED = 0xD4A6A7E0


@gin.configurable
def no_penalty():
  """reference penalty_lib.py:28-30."""
  return K.zeros(1)


def _slope_penalty(discriminator, points, y, is_training):
  """mean((sqrt(1e-4 + sum (d logits / d points)^2) - 1)^2) (penalty_lib.py:51-55, 76-81) through the taped double
  backward; `points` is a fresh leaf."""
  points.req = True                            # differentiate the logits wrt this leaf
  with tape.record(True):
    logits = discriminator(points, y=y, is_training=is_training, reuse=True)[1]
    ones = K.fill_(K.empty(*logits.shape), 1.0)
    (gradients,) = tape.backward([(logits, ones)], [points], K.add_grad, create_graph=True)
    return K.gp_penalty(gradients)


@gin.configurable(whitelist=[])
def dragan_penalty(discriminator, x, y, is_training, step=None):
  """DRAGAN gradient penalty (reference penalty_lib.py:33-57) at the real batch perturbed by std(x) * (U - 0.5) and
  clipped to [0, 1].  The moments run over this replica's whole batch (no collective, as on each TPU core).  U is drawn on
  the device from the counter-based stream at seed DRAGAN_SEED + replica id and offset step * numel(x), `step` being the
  discriminator's int32 step counter on the device (ModularGAN passes its Adam step before the update): every replay of
  a captured cycle draws fresh noise, and a restored snapshot or checkpoint continues the stream."""
  if step is None:
    raise ValueError("dragan_penalty needs the discriminator's device step counter (step=...) to key its noise")
  from ..tpu import tpu_ops
  x_noisy, _ = K.dragan_perturb(x, DRAGAN_SEED + tpu_ops.replica_id(), step)
  return _slope_penalty(discriminator, x_noisy, y, is_training)


@gin.configurable(whitelist=[])
def wgangp_penalty(discriminator, x, x_fake, y, is_training, alpha=None):
  """WGAN gradient penalty (reference penalty_lib.py:59-82).  `alpha` [B,1,1,1] may be fed (parity tests,
  bench); otherwise it is drawn U[0,1) on the device."""
  if alpha is None:
    # tf.random.uniform (penalty_lib.py:72-73) through the library's counter-based generator (cgan_random_uniform): no
    # torch op on the product path; successive draws advance the offset
    from ..tpu import tpu_ops
    alpha = K.empty(x.shape[0], 1, 1, 1)
    # every replica draws its own coefficients (the reference's per-replica tf.random.uniform): the rank selects the stream
    K._call("random_uniform", alpha.ptr, alpha.numel, _ALPHA_RNG["seed"] + tpu_ops.replica_id(), _ALPHA_RNG["offset"])
    _ALPHA_RNG["offset"] += alpha.numel
  return _slope_penalty(discriminator, K.interpolate(x, x_fake, alpha), y, is_training)


def l2_kernels(params):
  """The variables l2_penalty penalises among a network's trainable ones: those named `.../kernel` (the reference keeps
  `discriminator.trainable_variables` ending in `/kernel:0`), so no bias, gamma / beta, sigma or u_var."""
  return type(params)((k, v) for k, v in params.items() if k.endswith("/kernel"))


@gin.configurable(whitelist=[])
def l2_penalty(discriminator, kernel_segments=None):
  """L2 penalty (reference penalty_lib.py:85-103): the mean over D's kernels of sum(w^2) / 2.  `kernel_segments` is the
  K.KernelSegments of D's packed kernels (ModularGAN builds it when this penalty is bound); the gradient lands in the
  flat gradient buffer when the model calls its add_pending_grads(), before the gradient exchange."""
  del discriminator           # the variables come from kernel_segments, which the model selected with l2_kernels
  if kernel_segments is None:
    raise ValueError("l2_penalty needs the discriminator's packed kernel table (kernel_segments=...)")
  return K.l2_penalty(kernel_segments)


@gin.configurable("penalty", whitelist=["fn"])
def get_penalty_loss(fn=no_penalty, **kwargs):
  """Returns the penalty loss (reference penalty_lib.py:105-108)."""
  return utils.call_with_accepted_args(fn, **kwargs)


def bound_penalty():
  """The function `penalty.fn` is bound to (no_penalty when it is not bound)."""
  try:
    fn = gin.query_parameter("penalty.fn")
  except KeyError:
    return no_penalty
  return fn.resolve() if hasattr(fn, "resolve") else fn
