"""InfoGAN pair (reference architectures/infogan.py:35-100; Chen et al. 2016), the network of the MNIST / Fashion-MNIST
studies.  Generator: two dense layers (1024, then 128 channels at a quarter of the image side), two 4x4 stride-2
transposed convolutions (64 channels, then the colours), batch norm + leaky ReLU(0.2) in between, sigmoid.
Discriminator: two 4x4 stride-2 convolutions (64, 128), a dense layer of 1024 features and a dense logit, leaky ReLU(0.2)
throughout.

As in the reference, the generator calls `arch_ops.batch_norm` itself (`G.batch_norm_fn` does not reach it) and ignores
y; the discriminator normalises d_conv2 and d_fc3 with `D.batch_norm_fn` (the identity when it is unbound) and applies
`D.spectral_norm` to all four of its layers.  `D.layer_norm` is accepted and ignored."""
from .. import kernels as K
from . import abstract_arch
from . import arch_ops as ops
from . import netdef

KERNEL, STRIDE = 4, 2


class Generator(abstract_arch.AbstractGenerator):

  def apply(self, z, y, is_training):
    del y
    height, width, colors = self._image_shape
    flow = netdef.Flow(self, z)
    flow.linear(1024, "g_fc1").through(ops.batch_norm, is_training, name="g_bn1").lrelu()
    flow.linear(128 * (height // 4) * (width // 4), "g_fc2").through(ops.batch_norm, is_training, name="g_bn2")
    flow.lrelu(_tf32=True).reshape(z.shape[0], height // 4, width // 4, 128)
    flow.deconv((height // 2, width // 2), 64, KERNEL, STRIDE, "g_dc3")
    flow.through(ops.batch_norm, is_training, name="g_bn3").lrelu(_tf32=True)
    flow.deconv((height, width), colors, KERNEL, STRIDE, "g_dc4")
    return K.sigmoid(flow.x)


class Discriminator(abstract_arch.AbstractDiscriminator):

  def apply(self, x, y, is_training):
    sn = self._spectral_norm
    flow = netdef.Flow(self, x, y=y, is_training=is_training)
    flow.conv(64, KERNEL, STRIDE, "d_conv1", use_sn=sn).lrelu(_tf32=True)
    flow.conv(128, KERNEL, STRIDE, "d_conv2", use_sn=sn).norm("d_bn2").lrelu()
    flow.reshape(x.shape[0], -1).linear(1024, "d_fc3", use_sn=sn).norm("d_bn3").lrelu()
    features = flow.x
    logit = flow.linear(1, "d_fc4", use_sn=sn).x
    return K.sigmoid(logit), logit, features
