"""The four GAN objectives behind the reference's call surface (gans/loss_lib.py:30-154: `non_saturating`, `wasserstein`,
`least_squares`, `hinge`, `check_dimensions`, `get_losses`, gin name `loss.fn`).  All of them are ONE fused kernel here
(`cgan_gan_loss`: a warp-shuffle reduction over the [real; fake] logit vector that returns d_loss, d_loss_real,
d_loss_fake, g_loss and, on the backward pass, d(loss)/d(logit)); this module only validates shapes and selects the
kernel's `kind`."""
from .. import gin_lite as gin
from .. import kernels as K
from .. import utils


def check_dimensions(d_real, d_fake, d_real_logits, d_fake_logits):
  """Predictions and logits must pairwise agree in shape and be [batch, 1]-like rank-2 tensors."""
  pairs = ((d_real, d_fake), (d_real_logits, d_fake_logits), (d_real, d_real_logits))
  for first, second in pairs:
    if first is None or second is None:
      continue
    a, b = list(first.shape), list(second.shape)
    if a != b:
      raise ValueError("Shape mismatch: %s vs %s." % (a, b))
    if len(a) != 2 or len(b) != 2:
      raise ValueError("Rank: expected 2, got %s and %s" % (len(a), len(b)))


def _objective(kind, logits_first):
  """Builds the public function for `kind`.  The reference's signatures differ in which pair comes first (the least
  squares loss is defined on probabilities, the others on logits); callers pass keywords (`get_losses`), so both
  orders are kept."""
  def run(d_real, d_fake, d_real_logits, d_fake_logits):
    check_dimensions(d_real, d_fake, d_real_logits, d_fake_logits)
    if d_real_logits is None or d_fake_logits is None:
      raise ValueError("The loss kernel works from logits; pass d_real_logits and d_fake_logits.")
    return K.gan_losses(kind, d_real_logits, d_fake_logits)     # sigmoid(logits) is recomputed inside the kernel

  if logits_first:
    def loss(d_real_logits, d_fake_logits, d_real=None, d_fake=None):
      return run(d_real, d_fake, d_real_logits, d_fake_logits)
  else:
    def loss(d_real, d_fake, d_real_logits=None, d_fake_logits=None):
      return run(d_real, d_fake, d_real_logits, d_fake_logits)
  loss.__name__ = loss.__qualname__ = kind
  loss.__doc__ = "%s loss: (d_loss, d_loss_real, d_loss_fake, g_loss) as device scalars." % kind
  return gin.configurable(whitelist=[])(loss)


non_saturating = _objective("non_saturating", True)      # loss_lib.py:53-78
wasserstein = _objective("wasserstein", True)            # loss_lib.py:81-101
least_squares = _objective("least_squares", False)       # loss_lib.py:104-124
hinge = _objective("hinge", True)                        # loss_lib.py:127-148


@gin.configurable("loss", whitelist=["fn"])
def get_losses(fn=non_saturating, **kwargs):
  """The configured objective applied to whichever of (d_real, d_fake, d_real_logits, d_fake_logits) it accepts."""
  return utils.call_with_accepted_args(fn, **kwargs)
