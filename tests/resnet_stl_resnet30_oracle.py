"""TEST INFRASTRUCTURE ONLY: the resnet_stl and resnet30 pairs (reference architectures/resnet_stl.py:33-108,
resnet30.py:36-143) restated on the oracle's PyTorch-CPU ops.  Importing this module adds "resnet_stl_arch" and
"resnet30_arch" to the architecture tables of `oracle/nets.py`; the entries already there are left as they are.  Both
pairs read their base width from `cfg.ch` (the reference's value is 64).  Every block goes through
`onets.resnet_block` looked up at call time, so `layer_norm_oracle.discriminator_layer_norm()` applies to them."""
import torch

from oracle import nets as onets


def _gen_resnet_stl(store, cfg, z, y, is_training):
  """resnet_stl.Generator.apply: fc_noise to a 6x6 x 8ch seed, three up blocks, final_norm, ReLU, final_conv."""
  sn, bn, ch = cfg.g_sn, cfg.g_bn, cfg.ch
  widths = [8 * ch, 4 * ch, 2 * ch, ch]
  h = onets.linear(store, cfg, z, 6 * 6 * widths[0], "fc_noise").reshape(-1, 6, 6, widths[0])
  for i in range(3):
    h = onets.resnet_block(store, cfg, h, "B%d" % (i + 1), widths[i], widths[i + 1], "up", True, y, is_training, bn, sn)
  h = torch.relu(onets.apply_bn(store, cfg, bn, h, y, is_training, "final_norm", sn))
  h = onets.conv2d(store, cfg, h, cfg.image_shape[2], 3, 3, 1, "final_conv")
  return torch.sigmoid(h)


def _disc_resnet_stl(store, cfg, x, y, is_training):
  """resnet_stl.Discriminator.apply: B0-B3 down, B4 at the same size, ReLU, spatial mean, disc_final_fc."""
  sn, bn, ch = cfg.d_sn, cfg.d_bn, cfg.ch
  if x.dim() != 4 or x.shape[1] != x.shape[2]:
    raise ValueError("Input tensor must be a square rank-4 batch.")
  colors = x.shape[3]
  if colors not in (1, 3):
    raise ValueError("Number of color channels unknown: %s" % colors)
  widths = [colors, ch, 2 * ch, 4 * ch, 8 * ch, 16 * ch]
  h = x
  for i in range(5):
    h = onets.resnet_block(store, cfg, h, "B%d" % i, widths[i], widths[i + 1], "down" if i < 4 else "none", False, y,
                           is_training, bn, sn)
  feat = torch.relu(h).mean(dim=(1, 2))
  logit = onets.linear(store, cfg, feat, 1, "disc_final_fc", use_sn=sn)
  return torch.sigmoid(logit), logit, feat


def _gen_resnet30(store, cfg, z, y, is_training):
  """resnet30.Generator.apply: fc_noise to 4x4 x 8ch, six superblocks of five blocks (+ an up block in the first five,
  halving the width), final_conv straight after the last block."""
  sn, bn, ch = cfg.g_sn, cfg.g_bn, cfg.ch
  h = onets.linear(store, cfg, z, 4 * 4 * 8 * ch, "fc_noise").reshape(-1, 4, 4, 8 * ch)
  cin = 8 * ch
  for s in range(6):
    for i in range(5):
      h = onets.resnet_block(store, cfg, h, "B_%d_%d" % (s, i), cin, cin, "none", True, y, is_training, bn, sn)
    if s < 5:
      h = onets.resnet_block(store, cfg, h, "B_%d_up" % s, cin, cin // 2, "up", True, y, is_training, bn, sn)
    cin //= 2
  h = onets.conv2d(store, cfg, h, cfg.image_shape[2], 3, 3, 1, "final_conv")
  return torch.sigmoid(h)


def _disc_resnet30(store, cfg, x, y, is_training):
  """resnet30.Discriminator.apply: color_conv to ch/4, six superblocks (+ a down block named B_<s>_up in the first
  five, doubling the width), the last map flattened straight into disc_final_fc."""
  sn, bn, ch = cfg.d_sn, cfg.d_bn, cfg.ch
  side = x.shape[1]
  if x.dim() != 4 or x.shape[1] != x.shape[2] or side & (side - 1):
    raise ValueError("Input tensor must be a square rank-4 batch, a power of two wide.")
  if x.shape[3] not in (1, 3):
    raise ValueError("Number of color channels unknown: %s" % x.shape[3])
  h = onets.conv2d(store, cfg, x, ch // 4, 3, 3, 1, "color_conv")
  cin = ch // 4
  for s in range(6):
    for i in range(5):
      h = onets.resnet_block(store, cfg, h, "B_%d_%d" % (s, i), cin, cin, "none", False, y, is_training, bn, sn)
    if s < 5:
      h = onets.resnet_block(store, cfg, h, "B_%d_up" % s, cin, 2 * cin, "down", False, y, is_training, bn, sn)
    cin *= 2
  feat = h.reshape(x.shape[0], -1)
  logit = onets.linear(store, cfg, feat, 1, "disc_final_fc", use_sn=sn)
  return torch.sigmoid(logit), logit, feat


onets._GENS.setdefault("resnet_stl_arch", _gen_resnet_stl)
onets._GENS.setdefault("resnet30_arch", _gen_resnet30)
onets._DISCS.setdefault("resnet_stl_arch", _disc_resnet_stl)
onets._DISCS.setdefault("resnet30_arch", _disc_resnet30)
