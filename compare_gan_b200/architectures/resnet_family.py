"""The "plain" ResNet pairs (CIFAR 32x32, the five-block 128x128 one, the 48x48 STL one and the 30-block 128x128 one)
share everything but their tables: a dense seed, residual blocks, [BN-ReLU-]conv3x3-sigmoid on the generator side;
[a colour convolution,] residual blocks, then ReLU and spatial mean or a plain flatten, dense logit (+ optional class
projection) on the discriminator side.  The concrete modules (`resnet_cifar`, `resnet5`, `resnet_stl`, `resnet30`) only
provide a `GeneratorPlan` / `DiscriminatorPlan`; this module runs them."""
import collections

from .. import kernels as K
from . import arch_ops as ops
from . import netdef
from . import resnet_ops

SEED = 4

GeneratorPlan = collections.namedtuple(
    "GeneratorPlan", "widths scales hierarchical_z embed_z embed_y spectral_norm_outside_blocks seed names final_norm",
    defaults=(SEED, None, True))
# widths: seed width followed by each block's output width; scales: one of "up"/"none" per block;
# spectral_norm_outside_blocks: whether the dense seed, the embeddings and the final conv follow G.spectral_norm;
# seed: side of the dense seed map; names: block names (None: B1, B2, ...); final_norm: BN-ReLU before final_conv

DiscriminatorPlan = collections.namedtuple(
    "DiscriminatorPlan", "first_block widths scales project_y names color_conv flatten power_of_two",
    defaults=(None, None, False, True))
# first_block: index in the block names ("B0" or "B1"); widths: output width per block; scales: "down"/"none" per block;
# names: block names (None: B<first_block>, ...); color_conv: width of a 3x3 convolution (no spectral norm) in front of
# the blocks, or None; flatten: the features are the last block's output flattened (NHWC order) rather than the spatial
# mean of its ReLU; power_of_two: the input side must be a power of two


class PlainResNetGenerator(resnet_ops.ResNetGenerator):

  def _plan(self):
    raise NotImplementedError

  def apply(self, z, y, is_training):
    plan = self._plan()
    sn = self._spectral_norm and plan.spectral_norm_outside_blocks
    if plan.embed_z:
      z = ops.linear(z, z.shape[1], scope="embed_z", use_sn=sn)
    if plan.embed_y:
      y = ops.linear(y, z.shape[1], scope="embed_y", use_sn=sn)
    z_seed, z_blocks, y_blocks = netdef.split_latent(z, y, len(plan.scales), plan.hierarchical_z)
    flow = netdef.Flow(self, z_seed, z=z, y=y, is_training=is_training)
    flow.linear(plan.seed * plan.seed * plan.widths[0], "fc_noise", use_sn=sn).reshape(-1, plan.seed, plan.seed,
                                                                                        plan.widths[0])
    for i, scale in enumerate(plan.scales):
      name = plan.names[i] if plan.names else "B%d" % (i + 1)
      block = self._resnet_block(name, plan.widths[i], plan.widths[i + 1], scale)
      flow.x = block(flow.x, z=z_blocks[i], y=y_blocks[i], is_training=is_training)
    if plan.final_norm:
      flow.norm_relu("final_norm", tf32=True)
    flow.conv(self._image_shape[2], 3, 1, "final_conv", use_sn=sn)
    return K.sigmoid(flow.x)


class PlainResNetDiscriminator(resnet_ops.ResNetDiscriminator):

  def _plan(self, colors):
    raise NotImplementedError

  def apply(self, x, y, is_training):
    plan = self._plan(x.shape[-1])
    resnet_ops.validate_image_inputs(x, validate_power2=plan.power_of_two)
    colors = x.shape[3]
    if colors not in (1, 3):
      raise ValueError("Number of color channels not supported: {}".format(colors))
    net, width = x, colors
    if plan.color_conv:
      net, width = ops.conv2d(x, plan.color_conv, 3, 3, 1, 1, name="color_conv"), plan.color_conv
    for i, (out_width, scale) in enumerate(zip(plan.widths, plan.scales)):
      name = plan.names[i] if plan.names else "B%d" % (plan.first_block + i)
      block = self._resnet_block(name, width, out_width, scale)
      net, width = block(net, z=None, y=y, is_training=is_training), out_width
    if plan.flatten:
      features = K.reshape(net, net.shape[0], -1)
      width = features.shape[1]
    else:
      features = K.globalpool(K.relu(net), mean=True)
    logit = ops.linear(features, 1, scope="disc_final_fc", use_sn=self._spectral_norm)
    if plan.project_y:
      if y is None:
        raise ValueError("You must provide class information y to project.")
      embedded = ops.linear(y, width, use_bias=False, scope="embedding_fc", use_sn=self._spectral_norm)
      logit = K.add(logit, netdef.projection_term(embedded, features))
    return K.sigmoid(logit), logit, features
