"""Building material for the network definitions of this package.

The reference spells every network out imperatively in TensorFlow; here a network is a short table (channel plan, block
plan, layer list) that is *run* by the helpers below, which is what the CUDA-graph engine wants anyway: one place that
decides which fused kernel-layer call a (norm, activation, convolution, resampling) group turns into.

* `Flow`      — a running activation plus chainable layer calls (linear, conv, deconv, norm, activations, reshape).
* `BlockPlan` / `residual_block` — ONE pre-activation residual block covering both families the reference has
  (`resnet_ops.ResNetBlock`: 3x3 shortcut convolution evaluated first; `resnet_biggan.BigGanResNetBlock`: optional 1x1
  shortcut evaluated last).  Up-sampling is fused into the convolution's gather (`_upsample`), down-sampling is the 2x2
  average pool behind the convolution, ReLU is fused into the batch-norm apply kernel (`arch_ops.norm_relu`).
* `split_latent` — the "hierarchical z" routing shared by the CIFAR ResNet and BigGAN generators.
* `projection_term`, `halvings`, `check_square_power_of_two`.

Variable scopes and names are the reference's (they are the checkpoint key space, pinned by
`tests/test_arch_traces.py` against `architectures/resnet_norm_test.py`).
"""
import collections
import math

from .. import kernels as K
from .. import variables as V
from . import arch_ops as ops

SCALES = ("up", "down", "none")


def check_square_power_of_two(inputs, validate_power2=True):
  """Image batches must be rank 4, square and (optionally) a power of two wide (reference resnet_ops.py:59-67)."""
  if len(inputs.shape) != 4:
    raise ValueError("Input tensor must have rank 4.")
  side_h, side_w = inputs.shape[1], inputs.shape[2]
  if side_h != side_w:
    raise ValueError("Input tensor does not have equal width and height: ", inputs.shape[1:3])
  if validate_power2 and math.log(side_h, 2) != int(math.log(side_h, 2)):
    raise ValueError("Input tensor `width` is not a power of 2: ", side_h)


def halvings(height, width, levels):
  """[(h, w), (ceil(h/2), ceil(w/2)), ...]: the spatial pyramid of stride-2 SAME (transposed) convolutions."""
  out = [(height, width)]
  for _ in range(levels):
    height, width = -(-height // 2), -(-width // 2)
    out.append((height, width))
  return out


class Flow(object):
  """The activation flowing through a network definition; every method applies one layer and returns `self`."""

  def __init__(self, net, x, z=None, y=None, is_training=True):
    self.net, self.x = net, x
    self._norm_kw = dict(z=z, y=y, is_training=is_training)

  # -- parametrised layers (arch_ops) --
  def linear(self, units, scope, **kw):
    self.x = ops.linear(self.x, units, scope=scope, **kw)
    return self

  def conv(self, channels, kernel, stride, name, **kw):
    self.x = ops.conv2d(self.x, channels, kernel, kernel, stride, stride, name=name, **kw)
    return self

  def deconv(self, out_hw, channels, kernel, stride, name):
    shape = [self.x.shape[0], out_hw[0], out_hw[1], channels]
    self.x = ops.deconv2d(self.x, shape, kernel, kernel, stride, stride, name=name)
    return self

  # -- normalisation through the owning network's configured batch-norm function --
  def norm(self, name):
    self.x = self.net.batch_norm(self.x, name=name, **self._norm_kw)
    return self

  def norm_relu(self, name, tf32=False):
    """`tf32`: the next layer is a (transposed) convolution, see arch_ops.norm_relu."""
    self.x = ops.norm_relu(self.net.batch_norm, self.x, name=name, _tf32=tf32, **self._norm_kw)
    return self

  # -- pointwise / shape --
  def relu(self, tf32=False):
    self.x = K.relu(self.x, round_tf32=tf32)
    return self

  def lrelu(self, **kw):
    self.x = ops.lrelu(self.x, **kw)
    return self

  def reshape(self, *shape):
    self.x = K.reshape(self.x, *shape)
    return self

  def through(self, fn, *args, **kw):
    self.x = fn(self.x, *args, **kw)
    return self


BlockPlan = collections.namedtuple("BlockPlan", "name cin cout scale generator_side shortcut")
# shortcut: "conv3x3_first" (resnet_ops.ResNetBlock), "conv1x1_last" (BigGAN), None (BigGAN block with equal widths)


def _block_conv(x, plan, cin, cout, scale, suffix, kernel, use_sn, pool=True, **fused):
  """One convolution of a residual block.  `pool=False` leaves the 2x2 average pool of a down-sampling convolution to the
  caller (who applies it once to the sum of both branches); `fused` are arch_ops.conv2d's epilogue arguments."""
  if x.shape[-1] != cin:
    raise ValueError("Unexpected number of input channels.")
  if scale not in SCALES:
    raise ValueError("Scale: got {}, expected 'up', 'down', or 'none'.".format(scale))
  prefix = "same" if scale == "none" else scale
  y = ops.conv2d(x, output_dim=cout, k_h=kernel, k_w=kernel, d_h=1, d_w=1, use_sn=use_sn,
                 name="{}_{}".format(prefix, suffix), _upsample=(scale == "up"), **fused)
  return K.avgpool2(y) if (scale == "down" and pool) else y


def _norm_relu(batch_norm, layer_norm, x, idx, tf32, norm_kw):
  """bn<idx> [-> ln<idx>] -> relu (resnet_ops.py:162-174, resnet_biggan.py:123-134), the ReLU fused into the last
  normaliser."""
  if not layer_norm:
    return ops.norm_relu(batch_norm, x, name="bn" + idx, _tf32=tf32, **norm_kw)
  h = batch_norm(x, name="bn" + idx, **norm_kw)
  return ops.layer_norm(h, norm_kw["is_training"], "ln" + idx, _relu=True, _tf32=tf32)


def residual_block(inputs, plan, batch_norm, z, y, is_training, use_sn, layer_norm=False):
  """One recomputed segment (arch_ops.recomputed) of inputs, z and y: see _residual_block."""
  return ops.recomputed(lambda x, z_, y_: _residual_block(x, plan, batch_norm, z_, y_, is_training, use_sn, layer_norm),
                        inputs, z, y)


def _residual_block(inputs, plan, batch_norm, z, y, is_training, use_sn, layer_norm):
  """norm-relu-conv, norm-relu-conv plus the plan's shortcut.  A generator block resamples in its FIRST convolution, a
  discriminator block in its SECOND (reference resnet_ops.py:93-102).  `layer_norm` puts ln1 / ln2 behind bn1 / bn2
  (the `D.layer_norm` binding).

  What the reference runs as separate TF ops is folded into the convolutions' epilogues where that is exact:
  * the residual add is done by the LAST convolution evaluated (conv2 for the 3x3-shortcut family, the 1x1 shortcut for
    BigGAN's) — `_residual`;
  * a down-sampling block pools ONCE: avgpool(a) + avgpool(b) == avgpool(a + b), so both branches stay at full
    resolution until their sum;
  * without a normaliser between the two convolutions (a discriminator without layer norm) the second ReLU is conv1's
    epilogue;
  * every tensor whose only consumer is a tensor-core convolution is stored TF32-rounded (`_tf32`)."""
  if inputs.shape[-1] != plan.cin:
    if plan.shortcut == "conv3x3_first":
      raise ValueError("Unexpected number of input channels.")
    raise ValueError("Unexpected number of input channels (expected {}, got {}).".format(plan.cin, inputs.shape[-1]))
  first = plan.scale if plan.generator_side else "none"
  second = "none" if plan.generator_side else plan.scale
  norm_kw = dict(z=z, y=y, is_training=is_training)
  plain = ops.configured_norm(batch_norm) is None and not layer_norm     # no normaliser between the convolutions
  with V.variable_scope(plan.name):
    skip = None
    if plan.shortcut == "conv3x3_first":
      skip = _block_conv(inputs, plan, plan.cin, plan.cout, plan.scale, "conv_shortcut", 3, use_sn, pool=False)
    # (a block fed by the 3-channel image runs its first convolutions in the exact-fp32 streaming kernels: no rounding)
    h = _norm_relu(batch_norm, layer_norm, inputs, "1", plan.cin > 4, norm_kw)
    if plain and first != "down":
      h = _block_conv(h, plan, plan.cin, plan.cout, first, "conv1", 3, use_sn, _relu=True, _tf32=True)
    else:
      h = _block_conv(h, plan, plan.cin, plan.cout, first, "conv1", 3, use_sn)
      h = _norm_relu(batch_norm, layer_norm, h, "2", True, norm_kw)
    if plan.shortcut == "conv3x3_first":
      h = _block_conv(h, plan, plan.cout, plan.cout, second, "conv2", 3, use_sn, pool=False, _residual=skip)
      return ops.observe(K.avgpool2(h) if plan.scale == "down" else h)
    if plan.shortcut == "conv1x1_last" and plan.scale != "up":
      h = _block_conv(h, plan, plan.cout, plan.cout, second, "conv2", 3, use_sn, pool=False)
      h = _block_conv(inputs, plan, plan.cin, plan.cout, plan.scale, "conv_shortcut", 1, use_sn, pool=False, _residual=h)
      return ops.observe(K.avgpool2(h) if plan.scale == "down" else h)
    h = _block_conv(h, plan, plan.cout, plan.cout, second, "conv2", 3, use_sn)
    if plan.shortcut == "conv1x1_last":                      # 1x1 over a zero-inserted input: bias-only phases, plain add
      skip = _block_conv(inputs, plan, plan.cin, plan.cout, plan.scale, "conv_shortcut", 1, use_sn)
    return ops.observe(h if skip is None else K.add(h, skip))


def split_latent(z, y, num_blocks, hierarchical):
  """Returns (z for the seed layer, per-block z, per-block conditioning).  With `hierarchical` z is cut into
  num_blocks + 1 equal chunks: the first feeds the seed, chunk i (concatenated with y, if any) conditions block i."""
  if not hierarchical:
    return z, num_blocks * [z], num_blocks * [y]
  width = z.shape[1] // (num_blocks + 1)
  chunks = [K.slice_cols(z, i * width, (i + 1) * width) for i in range(num_blocks + 1)]
  per_block_y = num_blocks * [y] if y is None else [K.concat_cols(c, y) for c in chunks[1:]]
  return chunks[0], chunks[1:], per_block_y


def projection_term(embedded_y, features):
  """sum_c embed(y)_c * h_c, the projection-discriminator logit term (Miyato & Koyama; resnet_biggan.py:423)."""
  return K.rowdot(embedded_y, features)
