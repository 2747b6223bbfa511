"""Self-supervised GAN (reference gans/ssgan.py:40-226; Chen et al. 2018): ModularGAN plus a rotation-prediction head on
the discriminator's features.  The last `rotated_batch_size / 4` real and generated images of a sub-step are rotated by
90 / 180 / 270 degrees and appended to the discriminator batch; a linear head on the penultimate features classifies
the rotation; the discriminator learns it on real images (weight_rotation_loss_d), the generator is rewarded when its
samples are classifiable too (weight_rotation_loss_g).  Everything runs through the same taped C-ABI ops as ModularGAN
(`kernels.rot90`, `kernels.rotation_loss` are the two additions), so the cycle is captured into the same CUDA graph."""
from .. import gin_lite as gin
from .. import kernels as K
from .. import variables as V
from ..architectures import arch_ops as ops
from ..tpu import tpu_ops
from . import loss_lib, penalty_lib
from .modular_gan import ModularGAN

NUM_ROTATIONS = 4


def rotate_images(images, rot90_scalars=(0, 1, 2, 3)):
  """reference gans/utils.py:38-49: the requested rotations stacked along the batch axis."""
  out = None
  for k in rot90_scalars:
    r = K.rot90(images, k)
    out = r if out is None else K.concat_rows(out, r)
  return out


def _tile_rows(x, times):
  out = x
  for _ in range(times - 1):
    out = K.concat_rows(out, x)
  return out


@gin.configurable(blacklist=["dataset", "parameters", "model_dir"])
class SSGAN(ModularGAN):
  """Self-Supervised GAN, http://arxiv.org/abs/1811.11212 (reference gans/ssgan.py:40-84 constructor contract)."""

  def __init__(self, self_supervision="rotation_gan", rotated_batch_size=gin.REQUIRED, weight_rotation_loss_d=1.0,
               weight_rotation_loss_g=0.2, **kwargs):
    super(SSGAN, self).__init__(**kwargs)
    if rotated_batch_size is gin.REQUIRED:
      raise ValueError("SSGAN.rotated_batch_size is required")
    if self_supervision not in ("rotation_gan", "rotation_only", None, "none"):
      raise ValueError("Unknown self_supervision {}.".format(self_supervision))
    self._self_supervision = self_supervision or "none"
    self._rotated_batch_size = rotated_batch_size
    self._weight_rotation_loss_d = weight_rotation_loss_d
    self._weight_rotation_loss_g = weight_rotation_loss_g

  def discriminator_with_rotation_head(self, x, y, is_training):
    """reference :86-110 -> (probabilities, logits, rotation logits [N, 4])."""
    real_probs, real_scores, final = self.discriminator(x=x, y=y, is_training=is_training)
    use_sn = self.discriminator._spectral_norm
    with V.variable_scope("discriminator_rotation"):
      flat = K.reshape(final, x.shape[0], -1)
      rotation_scores = ops.linear(flat, NUM_ROTATIONS, scope="score_classify", use_sn=use_sn)
    return real_probs, real_scores, rotation_scores

  def _build_networks(self, f):
    """Variable creation pass: the rotation head's variables must exist before the flat packing."""
    gen, all_y = super(SSGAN, self)._build_networks(f)
    self.discriminator_with_rotation_head(K.concat_rows(f["images"], gen), y=all_y, is_training=True)
    return gen, all_y

  def create_loss(self, features, labels, params=None, is_training=True, for_discriminator=True):
    """reference :112-226.  As in ModularGAN.create_loss the penalty sub-graph only runs for the discriminator step."""
    images, generated = features["images"], features["generated"]
    if self.conditional:
      y = self._get_one_hot_labels(labels)
      sampled_y = self._get_one_hot_labels(features["sampled_labels"])
    else:
      y = sampled_y = None
    all_y = None
    bs = images.shape[0]
    num_replicas = tpu_ops.num_replicas()
    if self._rotated_batch_size % num_replicas != 0:
      raise ValueError("rotated_batch_size must be a multiple of the number of replicas")
    rotated_bs = self._rotated_batch_size // num_replicas
    if rotated_bs % 4 != 0:
      raise ValueError("rotated_batch_size per replica must be a multiple of 4")
    num_rotated_examples = rotated_bs // 4
    rotation = "rotation" in self._self_supervision
    if rotation:
      if num_rotated_examples > bs:
        raise ValueError("rotated_batch_size / 4 = %d exceeds the batch size %d" % (num_rotated_examples, bs))
      images_rotated = rotate_images(K.slice_rows(images, bs - num_rotated_examples, bs), rot90_scalars=(1, 2, 3))
      generated_rotated = rotate_images(K.slice_rows(generated, bs - num_rotated_examples, bs), rot90_scalars=(1, 2, 3))
      all_images = K.concat_rows(K.concat_rows(images, images_rotated), K.concat_rows(generated, generated_rotated))
      if self.conditional:
        y_rotated = _tile_rows(K.slice_rows(y, bs - num_rotated_examples, bs), 3)
        sampled_y_rotated = y_rotated          # the reference tiles y (not sampled_y) for both halves, ssgan.py:166-167
        all_y = K.concat_rows(K.concat_rows(y, y_rotated), K.concat_rows(sampled_y, sampled_y_rotated))
    else:
      all_images = K.concat_rows(images, generated)
      if self.conditional:
        all_y = K.concat_rows(y, sampled_y)
    d_all, d_all_logits, c_all_logits = self.discriminator_with_rotation_head(all_images, y=all_y, is_training=is_training)
    half = d_all.shape[0] // 2
    d_real, d_fake = K.slice_rows(d_all, 0, bs), K.slice_rows(d_all, half, half + bs)
    d_real_logits, d_fake_logits = K.slice_rows(d_all_logits, 0, bs), K.slice_rows(d_all_logits, half, half + bs)
    self.d_loss, _, _, self.g_loss = loss_lib.get_losses(
        d_real=d_real, d_fake=d_fake, d_real_logits=d_real_logits, d_fake_logits=d_fake_logits)
    if for_discriminator:
      penalty_loss = penalty_lib.get_penalty_loss(
          x=images, x_fake=generated, y=y, is_training=is_training, discriminator=self.discriminator,
          alpha=features.get("alpha"), step=self.d_opt.step, kernel_segments=self.d_kernels)
      self.penalty_loss = penalty_loss
      if penalty_loss.node is not None:
        self.d_loss = K.add(self.d_loss, K.affine(penalty_loss, self._lambda))
    if rotation:
      c_real_logits = K.slice_rows(c_all_logits, half - rotated_bs, half)        # the last rotated_bs rows of each half
      c_fake_logits = K.slice_rows(c_all_logits, 2 * half - rotated_bs, 2 * half)
      c_real_loss = K.rotation_loss(c_real_logits, NUM_ROTATIONS)
      c_fake_loss = K.rotation_loss(c_fake_logits, NUM_ROTATIONS)
      if self._self_supervision == "rotation_only":
        self.d_loss = K.affine(self.d_loss, 0.0)
        self.g_loss = K.affine(self.g_loss, 0.0)
      self.d_loss = K.add(self.d_loss, K.affine(c_real_loss, self._weight_rotation_loss_d))
      self.g_loss = K.add(self.g_loss, K.affine(c_fake_loss, self._weight_rotation_loss_g))
      self.c_real_loss, self.c_fake_loss = c_real_loss, c_fake_loss
