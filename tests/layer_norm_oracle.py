"""TEST INFRASTRUCTURE ONLY: the layer norm of `D.layer_norm = True` (reference arch_ops.py:448-450) on the oracle side.

`layer_norm` restates tf.contrib.layers.layer_norm op by op on PyTorch-CPU; torch autograd through it is the yard-stick of
the engine's layer-norm kernels, second order included.  `discriminator_layer_norm()` makes the oracle networks of
`oracle/nets.py` put it into their discriminator blocks — bn -> ln -> relu -> conv, as resnet_ops.py:162-173 and
resnet_biggan.py:123-134 do — by swapping in block functions that restate theirs with the two extra lines.  Pair it with
the engine binding `D.layer_norm = True` (BINDING)."""
import contextlib

import torch

from oracle import nets as onets

BINDING = "D.layer_norm = True"


def layer_norm(store, x, is_training, scope, stop_gradient=True):
  """tf.contrib.layers.layer_norm(x, trainable=is_training, scope=scope) with its defaults begin_norm_axis=1,
  begin_params_axis=-1: beta then gamma [C] (zeros / ones), moments per sample over every axis but the first.
  tf.nn.moments computes the variance as reduce_mean(squared_difference(x, stop_gradient(mean))): first-order
  gradients do not see the stop, the derivative of the backward (a gradient penalty) does, so torch autograd through
  this graph is TF's second order.  `stop_gradient=False` gives the exact Hessian instead (tests pin the difference)."""
  with store.scope(scope):
    c = x.shape[-1]
    beta = store.get("beta", (c,), ("zeros",), trainable=is_training)
    gamma = store.get("gamma", (c,), ("ones",), trainable=is_training)
  axes = tuple(range(1, x.dim()))
  mean = x.mean(dim=axes, keepdim=True)
  var = torch.square(x - (mean.detach() if stop_gradient else mean)).mean(dim=axes, keepdim=True)
  inv = torch.rsqrt(var + 1e-12) * gamma
  return x * inv + (beta - mean * inv)


def _resnet_block(store, cfg, x, name, cin, cout, scale, is_gen, y, is_training, bn, use_sn):
  """oracle.nets.resnet_block (resnet_ops.py:136-182) with ln1 / ln2 in discriminator blocks."""
  scale1 = scale if is_gen else "none"
  scale2 = "none" if is_gen else scale
  with store.scope(name):
    shortcut = onets._get_conv(store, cfg, x, cin, cout, scale, "conv_shortcut", use_sn)
    h = onets.apply_bn(store, cfg, bn, x, y, is_training, "bn1", use_sn)
    if not is_gen:
      h = layer_norm(store, h, is_training, "ln1")
    h = torch.relu(h)
    h = onets._get_conv(store, cfg, h, cin, cout, scale1, "conv1", use_sn)
    h = onets.apply_bn(store, cfg, bn, h, y, is_training, "bn2", use_sn)
    if not is_gen:
      h = layer_norm(store, h, is_training, "ln2")
    h = torch.relu(h)
    h = onets._get_conv(store, cfg, h, cout, cout, scale2, "conv2", use_sn)
    return onets._observe(store, h + shortcut)


def _biggan_block(store, cfg, x, name, cin, cout, scale, is_gen, y, is_training, bn, use_sn, add_shortcut=True):
  """oracle.nets.biggan_block (resnet_biggan.py:99-151) with ln1 / ln2 in discriminator blocks."""
  scale1 = scale if is_gen else "none"
  scale2 = "none" if is_gen else scale
  with store.scope(name):
    h = onets.apply_bn(store, cfg, bn, x, y, is_training, "bn1", use_sn)
    if not is_gen:
      h = layer_norm(store, h, is_training, "ln1")
    h = torch.relu(h)
    h = onets._get_conv(store, cfg, h, cin, cout, scale1, "conv1", use_sn)
    h = onets.apply_bn(store, cfg, bn, h, y, is_training, "bn2", use_sn)
    if not is_gen:
      h = layer_norm(store, h, is_training, "ln2")
    h = torch.relu(h)
    h = onets._get_conv(store, cfg, h, cout, cout, scale2, "conv2", use_sn)
    if add_shortcut:
      h = h + onets._get_conv(store, cfg, x, cin, cout, scale, "conv_shortcut", use_sn, ksize=1)
    return onets._observe(store, h)


@contextlib.contextmanager
def discriminator_layer_norm():
  """Inside this scope the oracle's resnet_cifar / resnet5 / resnet_biggan discriminators are layer-normalised (the
  other architectures never read the flag, as in the reference)."""
  saved = onets.resnet_block, onets.biggan_block
  onets.resnet_block, onets.biggan_block = _resnet_block, _biggan_block
  try:
    yield
  finally:
    onets.resnet_block, onets.biggan_block = saved
