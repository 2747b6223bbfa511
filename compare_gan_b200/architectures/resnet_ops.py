"""The classic pre-activation ResNet block family (reference architectures/resnet_ops.py:35-219) on top of
`netdef.residual_block`: a 3x3 shortcut convolution that is evaluated before the residual branch, up-sampling in the
first convolution of generator blocks and average-pool down-sampling behind the second convolution of discriminator
blocks.  `unpool` itself (resnet_ops.py:35-56) never materialises here — see `kernels.conv2d(upsample=True)`."""
from . import abstract_arch
from . import netdef

validate_image_inputs = netdef.check_square_power_of_two


class ResNetBlock(object):
  """A configured residual block; calling it applies it.  Subclass hook: `_shortcut_kind()`."""

  def __init__(self, name, in_channels, out_channels, scale, is_gen_block, layer_norm=False, spectral_norm=False,
               batch_norm=None):
    assert scale in netdef.SCALES
    self._in_channels, self._out_channels = in_channels, out_channels
    self._name, self._scale, self._is_gen_block = name, scale, is_gen_block
    self._layer_norm, self._spectral_norm = layer_norm, spectral_norm
    self.batch_norm = batch_norm

  def _shortcut_kind(self):
    return "conv3x3_first"

  def plan(self):
    return netdef.BlockPlan(self._name, self._in_channels, self._out_channels, self._scale, self._is_gen_block,
                            self._shortcut_kind())

  def apply(self, inputs, z, y, is_training):
    return netdef.residual_block(inputs, self.plan(), self.batch_norm, z, y, is_training, self._spectral_norm,
                                 layer_norm=self._layer_norm)

  __call__ = apply


def _block_factory(block_cls, allowed, side, **fixed):
  def make(self, name, in_channels, out_channels, scale, **extra):
    if scale not in allowed:
      raise ValueError("Unknown {} ResNet block scaling: {}.".format(side, scale))
    kw = dict(fixed, **extra)
    if side == "discriminator":
      kw["layer_norm"] = self._layer_norm
    return block_cls(name=name, in_channels=in_channels, out_channels=out_channels, scale=scale,
                     spectral_norm=self._spectral_norm, batch_norm=self.batch_norm, **kw)
  return make


class ResNetGenerator(abstract_arch.AbstractGenerator):
  """Generators made of up-sampling residual blocks (reference resnet_ops.py:185-200)."""
  _resnet_block = _block_factory(ResNetBlock, ("up", "none"), "generator", is_gen_block=True)


class ResNetDiscriminator(abstract_arch.AbstractDiscriminator):
  """Discriminators made of down-sampling residual blocks (reference resnet_ops.py:203-219)."""
  _resnet_block = _block_factory(ResNetBlock, ("down", "none"), "discriminator", is_gen_block=False)
