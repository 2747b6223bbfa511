"""TEST INFRASTRUCTURE ONLY: the infogan pair (reference architectures/infogan.py:35-100) restated on the oracle's
PyTorch-CPU ops, which run in the oracle's dtype (float64 for the yard-stick twins of tests/gpu_util.make_pair).
Importing this module adds "infogan_arch" to the architecture tables of `oracle/nets.py`; the entries already there are
left as they are.  As in the reference, G always applies plain batch norm (cfg.g_bn does not reach it) and ignores y;
D normalises with cfg.d_bn (None: the identity) and applies cfg.d_sn to all four layers."""
import torch

from oracle import nets as onets
from oracle import tf_ops as T


def _gen_infogan(store, cfg, z, y, is_training):
  """infogan.Generator.apply: g_fc1 1024, g_fc2 128 x (h/4) x (w/4), g_dc3 64, g_dc4 colours, sigmoid."""
  del y
  h, w, c = cfg.image_shape
  b = z.shape[0]
  net = onets.linear(store, cfg, z, 1024, "g_fc1")
  net = T.lrelu(onets.batch_norm(store, cfg, net, is_training, name="g_bn1"))
  net = onets.linear(store, cfg, net, 128 * (h // 4) * (w // 4), "g_fc2")
  net = T.lrelu(onets.batch_norm(store, cfg, net, is_training, name="g_bn2"))
  net = net.reshape(b, h // 4, w // 4, 128)
  net = onets.deconv2d(store, cfg, net, (b, h // 2, w // 2, 64), 4, 4, 2, "g_dc3")
  net = T.lrelu(onets.batch_norm(store, cfg, net, is_training, name="g_bn3"))
  net = onets.deconv2d(store, cfg, net, (b, h, w, c), 4, 4, 2, "g_dc4")
  return torch.sigmoid(net)


def _disc_infogan(store, cfg, x, y, is_training):
  """infogan.Discriminator.apply: d_conv1 64, d_conv2 128 + d_bn2, d_fc3 1024 + d_bn3, d_fc4; returns the 1024
  features after their leaky ReLU."""
  sn, bn = cfg.d_sn, cfg.d_bn
  net = T.lrelu(onets.conv2d(store, cfg, x, 64, 4, 4, 2, "d_conv1", use_sn=sn))
  net = onets.conv2d(store, cfg, net, 128, 4, 4, 2, "d_conv2", use_sn=sn)
  net = T.lrelu(onets.apply_bn(store, cfg, bn, net, y, is_training, "d_bn2", sn))
  net = net.reshape(x.shape[0], -1)
  net = onets.linear(store, cfg, net, 1024, "d_fc3", use_sn=sn)
  net = T.lrelu(onets.apply_bn(store, cfg, bn, net, y, is_training, "d_bn3", sn))
  logit = onets.linear(store, cfg, net, 1, "d_fc4", use_sn=sn)
  return torch.sigmoid(logit), logit, net


onets._GENS.setdefault("infogan_arch", _gen_infogan)
onets._DISCS.setdefault("infogan_arch", _disc_infogan)
