"""BigGAN networks for 32..512 pixels (reference architectures/resnet_biggan.py:80-425; Brock et al. 2018) as tables:
a channel plan per resolution, one residual-block family (1x1 shortcut, evaluated last, dropped in the discriminator
when the widths agree), the non-local block after the named blocks, hierarchical z + class embedding feeding every
conditional batch norm, projection discriminator.  All convolutions / matmuls dispatch to the tensor-core kernels through
`arch_ops`."""
from .. import gin_lite as gin
from .. import kernels as K
from .. import variables as V
from . import abstract_arch
from . import arch_ops as ops
from . import netdef
from . import resnet_ops

SEED_SIZE = 4
# channel multipliers along the network, by image resolution (generator: seed -> image; discriminator: image -> logit)
G_WIDTHS = {512: (16, 16, 8, 8, 4, 2, 1, 1), 256: (16, 16, 8, 8, 4, 2, 1), 128: (16, 16, 8, 4, 2, 1),
            64: (16, 16, 8, 4, 2), 32: (4, 4, 4, 4)}
D_WIDTHS = {512: (1, 1, 2, 4, 8, 8, 16, 16), 256: (1, 2, 4, 8, 8, 16, 16), 128: (1, 2, 4, 8, 16, 16),
            64: (2, 4, 8, 16, 16), 32: (2, 2, 2, 2)}


def _widths(table, resolution, ch):
  if resolution not in table:
    raise ValueError("Unsupported resolution: {}".format(resolution))
  return [ch * m for m in table[resolution]]


@gin.configurable
class BigGanResNetBlock(resnet_ops.ResNetBlock):
  """Residual block whose shortcut is a 1x1 convolution applied after the residual branch, or absent."""

  def __init__(self, add_shortcut=True, **kwargs):
    super(BigGanResNetBlock, self).__init__(**kwargs)
    self._add_shortcut = add_shortcut

  def _shortcut_kind(self):
    return "conv1x1_last" if self._add_shortcut else None


class _AttentionMixin(object):
  """`blocks_with_attention`: comma-separated block names that are followed by the non-local block."""

  def _after_block(self, name, net):
    if name in self._blocks_with_attention:
      net = ops.non_local_block(net, "non_local_block", use_sn=self._spectral_norm)
    return net


@gin.configurable
class Generator(_AttentionMixin, abstract_arch.AbstractGenerator):
  """seed 4x4 -> one up-sampling block per octave -> BN, ReLU, 3x3 conv, (tanh + 1) / 2."""

  def __init__(self, ch=96, blocks_with_attention="B4", hierarchical_z=True, embed_z=False, embed_y=True,
               embed_y_dim=128, embed_bias=False, **kwargs):
    super(Generator, self).__init__(**kwargs)
    self._ch, self._blocks_with_attention = ch, set(blocks_with_attention.split(","))
    self._hierarchical_z, self._embed_z = hierarchical_z, embed_z
    self._embed_y, self._embed_y_dim, self._embed_bias = embed_y, embed_y_dim, embed_bias

  _resnet_block = resnet_ops._block_factory(BigGanResNetBlock, ("up", "none"), "generator", is_gen_block=True)

  def _get_in_out_channels(self):
    widths = _widths(G_WIDTHS, self._image_shape[0], self._ch)
    return widths[:-1], widths[1:]

  def apply(self, z, y, is_training):
    cin, cout = self._get_in_out_channels()
    if self._embed_z:
      z = ops.linear(z, z.shape[1], scope="embed_z", use_sn=False, use_bias=self._embed_bias)
    if self._embed_y:
      y = ops.linear(y, self._embed_y_dim, scope="embed_y", use_sn=False, use_bias=self._embed_bias)
    z_seed, z_blocks, y_blocks = netdef.split_latent(z, y, len(cin), self._hierarchical_z)
    flow = netdef.Flow(self, z_seed, is_training=is_training)
    flow.linear(cin[0] * SEED_SIZE * SEED_SIZE, "fc_noise", use_sn=self._spectral_norm)
    flow.reshape(-1, SEED_SIZE, SEED_SIZE, cin[0])
    for i, (a, b) in enumerate(zip(cin, cout)):
      name = "B%d" % (i + 1)
      block = self._resnet_block(name, a, b, "up")
      flow.x = self._after_block(name, block(flow.x, z=z_blocks[i], y=y_blocks[i], is_training=is_training))
    flow.through(ops.batch_norm, is_training=is_training, name="final_norm", _relu=True, _tf32=True)
    flow.conv(self._image_shape[2], 3, 1, "final_conv", use_sn=self._spectral_norm)
    return K.tanh01(flow.x)


@gin.configurable
class Discriminator(_AttentionMixin, abstract_arch.AbstractDiscriminator):
  """one down-sampling block per octave (the last keeps the resolution) -> ReLU -> sum over space -> linear logit,
  plus the projection of the class embedding onto the pooled features."""

  def __init__(self, ch=96, blocks_with_attention="B1", project_y=True, **kwargs):
    super(Discriminator, self).__init__(**kwargs)
    self._ch, self._blocks_with_attention, self._project_y = ch, set(blocks_with_attention.split(",")), project_y

  _make_block = resnet_ops._block_factory(BigGanResNetBlock, ("down", "none"), "discriminator", is_gen_block=False)

  def _resnet_block(self, name, in_channels, out_channels, scale):
    return self._make_block(name, in_channels, out_channels, scale, add_shortcut=in_channels != out_channels)

  def _get_in_out_channels(self, colors, resolution):
    if colors not in (1, 3):
      raise ValueError("Unsupported color channels: {}".format(colors))
    widths = _widths(D_WIDTHS, resolution, self._ch)
    return [colors] + widths[:-1], widths

  def apply(self, x, y, is_training):
    resnet_ops.validate_image_inputs(x)
    cin, cout = self._get_in_out_channels(colors=x.shape[-1], resolution=x.shape[1])
    net = x
    for i, (a, b) in enumerate(zip(cin, cout)):
      name = "B%d" % (i + 1)
      block = self._resnet_block(name, a, b, "down" if i + 1 < len(cin) else "none")
      net = self._after_block(name, block(net, z=None, y=y, is_training=is_training))
    features = K.globalpool(K.relu(net), mean=False)
    logit = ops.linear(features, 1, scope="final_fc", use_sn=self._spectral_norm)
    if self._project_y:
      if y is None:
        raise ValueError("You must provide class information y to project.")
      with V.variable_scope("embedding_fc"):
        table = V.get_variable("kernel", (y.shape[1], cout[-1]), ops.glorot_normal)
        if self._spectral_norm:
          table = ops.spectral_norm(table)
        logit = K.add(logit, netdef.projection_term(K.matmul(y, table), features))
    return K.sigmoid(logit), logit, features
