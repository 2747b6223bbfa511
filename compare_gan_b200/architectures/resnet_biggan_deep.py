"""BigGAN-deep for 32..512 pixels (reference architectures/resnet_biggan_deep.py:61-434; Brock et al. 2018, appendix B):
twice as many residual blocks as BigGAN, each a bottleneck (1x1 -> 3x3 -> 3x3 -> 1x1 at a quarter of the wider end)
around an identity-preserving shortcut — channels are dropped on the way up and appended by a 1x1 convolution on the
way down; z is not chunked (every conditional batch norm sees [z, embed(y)]); attention sits at 64x64.  Expressed as
width tables + one block runner over `arch_ops`."""
from .. import gin_lite as gin
from .. import kernels as K
from .. import variables as V
from . import abstract_arch
from . import arch_ops as ops
from . import netdef
from . import resnet_ops

SEED_SIZE = 4
ATTENTION_RESOLUTION = 64
G_WIDTHS = {512: 4 * (16,) + 4 * (8,) + (4, 4, 2, 2, 1, 1, 1), 256: 4 * (16,) + 4 * (8,) + (4, 4, 2, 2, 1),
            128: 4 * (16,) + 2 * (8,) + (4, 4, 2, 2, 1), 64: 4 * (16,) + 2 * (8,) + (4, 4, 2), 32: 8 * (4,)}
D_WIDTHS = {512: (1, 1, 1, 2, 2, 4, 4) + 4 * (8,) + 4 * (16,), 256: (1, 2, 2, 4, 4) + 4 * (8,) + 4 * (16,),
            128: (1, 2, 2, 4, 4) + 2 * (8,) + 4 * (16,), 64: (2, 4, 4) + 2 * (8,) + 4 * (16,), 32: 8 * (2,)}
# (variable scope, kernel size, "mid" or "out" width, resampling this stage performs when the block's scale asks for it)
BOTTLENECK = (("conv1", 1, "mid", None), ("conv2", 3, "mid", "up"), ("conv3", 3, "mid", None), ("conv4", 1, "out", "down"))


def _channels(x):
  return x.shape[-1]


def _take_channels(x, count):
  n, h, w, c = x.shape
  return K.reshape(K.slice_cols(K.reshape(x, -1, c), 0, count), n, h, w, count)


def _append_channels(x, extra):
  n, h, w, c = x.shape
  both = K.concat_cols(K.reshape(x, -1, c), K.reshape(extra, -1, _channels(extra)))
  return K.reshape(both, n, h, w, c + _channels(extra))


@gin.configurable
class BigGanDeepResNetBlock(object):
  """Bottleneck residual block with an identity-preserving skip connection."""

  def __init__(self, name, in_channels, out_channels, scale, spectral_norm=False, batch_norm=None):
    assert scale in netdef.SCALES
    self._name, self._scale = name, scale
    self._in_channels, self._out_channels = in_channels, out_channels
    self._spectral_norm, self.batch_norm = spectral_norm, batch_norm

  def _shortcut(self, inputs):
    cin, cout, sn = self._in_channels, self._out_channels, self._spectral_norm
    with V.variable_scope("shortcut"):
      skip = inputs
      if cin > cout:
        assert self._scale == "up"
        skip = _take_channels(skip, cout)                    # drop the surplus channels
      if self._scale == "up":
        skip = K.unpool(skip)
      if self._scale == "down":
        skip = K.avgpool2(skip)
      if cin < cout:
        assert self._scale == "down"
        skip = _append_channels(skip, ops.conv1x1(skip, cout - cin, name="add_channels", use_sn=sn))
      return skip

  def apply(self, inputs, z, y, is_training):
    """One recomputed segment (arch_ops.recomputed) of inputs, z and y."""
    return ops.recomputed(lambda x, z_, y_: self._apply(x, z_, y_, is_training), inputs, z, y)

  def _apply(self, inputs, z, y, is_training):
    if _channels(inputs) != self._in_channels:
      raise ValueError("Unexpected number of input channels (expected {}, got {}).".format(
          self._in_channels, _channels(inputs)))
    widths = {"mid": max(self._in_channels, self._out_channels) // 4, "out": self._out_channels}
    with V.variable_scope(self._name):
      h = inputs
      for scope, kernel, width, resample in BOTTLENECK:
        active = resample == self._scale
        with V.variable_scope(scope):
          h = ops.norm_relu(self.batch_norm, h, z=z, y=y, is_training=is_training, name="bn",
                            _tf32=not (active and resample == "down"))
          if active and resample == "down":
            h = K.avgpool2(h)                                 # pooling precedes the closing 1x1 convolution
          h = ops.conv2d(h, widths[width], kernel, kernel, 1, 1, name="%dx%d_conv" % (kernel, kernel),
                         use_sn=self._spectral_norm, _upsample=active and resample == "up")
      return K.add(h, self._shortcut(inputs))

  __call__ = apply


def _plan(table, resolution, ch):
  if resolution not in table:
    raise ValueError("Unsupported resolution: {}".format(resolution))
  widths = [ch * m for m in table[resolution]]
  return list(zip(widths[:-1], widths[1:]))


@gin.configurable
class Generator(abstract_arch.AbstractGenerator):

  def __init__(self, ch=128, embed_y=True, embed_y_dim=128, experimental_fast_conv_to_rgb=False, **kwargs):
    super(Generator, self).__init__(**kwargs)
    if experimental_fast_conv_to_rgb:
      raise NotImplementedError("experimental_fast_conv_to_rgb is a TPU layout trick; the final conv is a thin tensor-core tile here")
    self._ch, self._embed_y, self._embed_y_dim = ch, embed_y, embed_y_dim

  def _resnet_block(self, name, in_channels, out_channels, scale):
    if scale not in ("up", "none"):
      raise ValueError("Unknown generator ResNet block scaling: {}.".format(scale))
    return BigGanDeepResNetBlock(name=name, in_channels=in_channels, out_channels=out_channels, scale=scale,
                                 spectral_norm=self._spectral_norm, batch_norm=self.batch_norm)

  def apply(self, z, y, is_training):
    plan = _plan(G_WIDTHS, self._image_shape[0], self._ch)
    if self._embed_y:
      y = ops.linear(y, self._embed_y_dim, scope="embed_y", use_sn=False, use_bias=False)
    if y is not None:
      y = K.concat_cols(z, y)
      z = y
    flow = netdef.Flow(self, z, is_training=is_training)
    flow.linear(plan[0][0] * SEED_SIZE * SEED_SIZE, "fc_noise", use_sn=self._spectral_norm)
    flow.reshape(-1, SEED_SIZE, SEED_SIZE, plan[0][0])
    for i, (cin, cout) in enumerate(plan):
      scale = "up" if i % 2 else "none"
      flow.x = self._resnet_block("B%d" % (i + 1), cin, cout, scale)(flow.x, z=z, y=y, is_training=is_training)
      if scale == "up" and flow.x.shape[1] == ATTENTION_RESOLUTION:
        flow.through(ops.non_local_block, "non_local_block", use_sn=self._spectral_norm)
    flow.through(ops.batch_norm, is_training=is_training, name="final_norm", _relu=True, _tf32=True)
    flow.conv(self._image_shape[2], 3, 1, "final_conv", use_sn=self._spectral_norm)
    return K.tanh01(flow.x)


@gin.configurable
class Discriminator(abstract_arch.AbstractDiscriminator):

  def __init__(self, ch=128, blocks_with_attention="B1", project_y=True, **kwargs):
    super(Discriminator, self).__init__(**kwargs)
    self._ch, self._project_y = ch, project_y
    self._blocks_with_attention = set(blocks_with_attention.split(","))     # kept for gin; placement is by resolution

  def _resnet_block(self, name, in_channels, out_channels, scale):
    if scale not in ("down", "none"):
      raise ValueError("Unknown discriminator ResNet block scaling: {}.".format(scale))
    return BigGanDeepResNetBlock(name=name, in_channels=in_channels, out_channels=out_channels, scale=scale,
                                 spectral_norm=self._spectral_norm, batch_norm=self.batch_norm)

  def apply(self, x, y, is_training):
    resnet_ops.validate_image_inputs(x)
    if _channels(x) not in (1, 3):
      raise ValueError("Unsupported color channels: {}".format(_channels(x)))
    plan = _plan(D_WIDTHS, x.shape[1], self._ch)
    sn = self._spectral_norm
    net = ops.conv2d(x, plan[0][0], 3, 3, 1, 1, name="initial_conv", use_sn=sn)
    for i, (cin, cout) in enumerate(plan):
      scale = "none" if i % 2 else "down"
      net = self._resnet_block("B%d" % (i + 1), cin, cout, scale)(net, z=None, y=y, is_training=is_training)
      if scale == "none" and net.shape[1] == ATTENTION_RESOLUTION:
        net = ops.non_local_block(net, "non_local_block", use_sn=sn)
    features = K.globalpool(K.relu(net), mean=False)
    logit = ops.linear(features, 1, scope="final_fc", use_sn=sn)
    if self._project_y:
      if y is None:
        raise ValueError("You must provide class information y to project.")
      with V.variable_scope("embedding_fc"):
        table = V.get_variable("kernel", (y.shape[1], plan[-1][1]), ops.glorot_normal)
        if sn:
          table = ops.spectral_norm(table)
        logit = K.add(logit, netdef.projection_term(K.matmul(y, table), features))
    return K.sigmoid(logit), logit, features
