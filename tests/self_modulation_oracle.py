"""TEST INFRASTRUCTURE ONLY: self-modulated batch norm (reference arch_ops.py:370-420) on the oracle side.

`self_modulated_batch_norm` restates the reference op on PyTorch-CPU.  Inside `self_modulated_generators()`, an oracle
network whose Cfg has `self_modulated = True` uses it in every generator normalisation the reference routes through
`self.batch_norm`: the scope swaps in generator functions that restate those of `oracle/nets.py` with z threaded to each
normaliser as the reference threads it (the per-block chunk under hierarchical z, the full, possibly embedded, z at
`final_norm`, [z, embed(y)] in BigGAN-deep).  They read `cfg.sbn_hidden` (num_hidden, default 32) and, for
resnet_cifar, `cfg.hierarchical_z`, `cfg.embed_z` and `cfg.embed_y`; other Cfgs run the oracle's own generators.  Pair
it with the engine binding `G.batch_norm_fn = @self_modulated_batch_norm`."""
import contextlib

import numpy as np
import torch

from oracle import nets as onets
from oracle import tf_ops as T


def self_modulated_batch_norm(store, cfg, x, z, is_training, use_sn, name="batch_norm"):
  """arch_ops.py:370-420: BN state first, then sbn/hidden, sbn/gamma (bias starting at 1), sbn/beta; h = z when
  num_hidden = 0."""
  if z is None:
    raise ValueError("You must provide z for self modulation.")
  hidden = getattr(cfg, "sbn_hidden", 32)
  with store.scope(name):
    out = onets.standardize_batch(store, cfg, x, is_training)
    c = x.shape[-1]
    shape = (-1, 1, 1, c) if x.dim() == 4 else (-1, c)
    with store.scope("sbn"):
      h = z
      if hidden > 0:
        h = torch.relu(onets.linear(store, cfg, h, hidden, "hidden", use_sn=use_sn))
      out = out * onets.linear(store, cfg, h, c, "gamma", use_sn=use_sn, bias_start=1.0).reshape(shape)
      return out + onets.linear(store, cfg, h, c, "beta", use_sn=use_sn).reshape(shape)


def _bn(store, cfg, x, z, is_training, name, use_sn):
  return self_modulated_batch_norm(store, cfg, x, z, is_training, use_sn, name=name)


def _resnet_block(store, cfg, x, name, cin, cout, scale, z, is_training, use_sn):
  """oracle.nets.resnet_block (resnet_ops.py:136-182), generator side."""
  with store.scope(name):
    shortcut = onets._get_conv(store, cfg, x, cin, cout, scale, "conv_shortcut", use_sn)
    h = torch.relu(_bn(store, cfg, x, z, is_training, "bn1", use_sn))
    h = onets._get_conv(store, cfg, h, cin, cout, scale, "conv1", use_sn)
    h = torch.relu(_bn(store, cfg, h, z, is_training, "bn2", use_sn))
    h = onets._get_conv(store, cfg, h, cout, cout, "none", "conv2", use_sn)
    return onets._observe(store, h + shortcut)


def _biggan_block(store, cfg, x, name, cin, cout, z, is_training, use_sn):
  """oracle.nets.biggan_block (resnet_biggan.py:99-151), up-sampling generator block."""
  with store.scope(name):
    h = torch.relu(_bn(store, cfg, x, z, is_training, "bn1", use_sn))
    h = onets._get_conv(store, cfg, h, cin, cout, "up", "conv1", use_sn)
    h = torch.relu(_bn(store, cfg, h, z, is_training, "bn2", use_sn))
    h = onets._get_conv(store, cfg, h, cout, cout, "none", "conv2", use_sn)
    h = h + onets._get_conv(store, cfg, x, cin, cout, "up", "conv_shortcut", use_sn, ksize=1)
    return onets._observe(store, h)


def _biggan_deep_block(store, cfg, x, name, cin, cout, scale, z, is_training, use_sn):
  """oracle.nets.biggan_deep_block (resnet_biggan_deep.py:61-177), generator side."""
  mid = max(cin, cout) // 4
  with store.scope(name):
    h = x
    with store.scope("conv1"):
      h = torch.relu(_bn(store, cfg, h, z, is_training, "bn", use_sn))
      h = onets.conv2d(store, cfg, h, mid, 1, 1, 1, "1x1_conv", use_sn)
    with store.scope("conv2"):
      h = torch.relu(_bn(store, cfg, h, z, is_training, "bn", use_sn))
      if scale == "up":
        h = T.unpool(h)
      h = onets.conv2d(store, cfg, h, mid, 3, 3, 1, "3x3_conv", use_sn)
    with store.scope("conv3"):
      h = torch.relu(_bn(store, cfg, h, z, is_training, "bn", use_sn))
      h = onets.conv2d(store, cfg, h, mid, 3, 3, 1, "3x3_conv", use_sn)
    with store.scope("conv4"):
      h = torch.relu(_bn(store, cfg, h, z, is_training, "bn", use_sn))
      h = onets.conv2d(store, cfg, h, cout, 1, 1, 1, "1x1_conv", use_sn)
    with store.scope("shortcut"):
      sc = x[..., :cout] if cin > cout else x
      if scale == "up":
        sc = T.unpool(sc)
    return h + sc


def _gen_resnet_cifar(store, cfg, z, y, is_training):
  """resnet_cifar.Generator.apply (resnet_cifar.py:58-112), hierarchical_z / embed_z / embed_y included."""
  sn = cfg.g_sn
  z_dim = z.shape[1]
  if getattr(cfg, "embed_z", False):
    z = onets.linear(store, cfg, z, z_dim, "embed_z", use_sn=sn)
  if cfg.embed_y:
    y = onets.linear(store, cfg, y, z_dim, "embed_y", use_sn=sn)
  if cfg.hierarchical_z:
    chunks = torch.chunk(z, 4, dim=1)
    z0, z_per_block = chunks[0], chunks[1:]
  else:
    z0, z_per_block = z, 3 * [z]
  h = onets.linear(store, cfg, z0, 4 * 4 * 256, "fc_noise", use_sn=sn).reshape(-1, 4, 4, 256)
  for i in range(3):
    h = _resnet_block(store, cfg, h, "B%d" % (i + 1), 256, 256, "up", z_per_block[i], is_training, sn)
  h = torch.relu(_bn(store, cfg, h, z, is_training, "final_norm", sn))
  return torch.sigmoid(onets.conv2d(store, cfg, h, cfg.image_shape[2], 3, 3, 1, "final_conv", use_sn=sn))


def _gen_resnet5(store, cfg, z, y, is_training, ch=64, channels=(8, 8, 4, 4, 2, 1)):
  """resnet5.Generator.apply (resnet5.py:45-93)."""
  sn = cfg.g_sn
  up_layers = int(np.log2(float(cfg.image_shape[0]) / 4))
  h = onets.linear(store, cfg, z, ch * channels[0] * 16, "fc_noise").reshape(-1, 4, 4, ch * channels[0])
  for i in range(5):
    h = _resnet_block(store, cfg, h, "B%d" % (i + 1), ch * channels[i], ch * channels[i + 1],
                      "up" if i < up_layers else "none", z, is_training, sn)
  h = torch.relu(_bn(store, cfg, h, z, is_training, "final_norm", sn))
  return torch.sigmoid(onets.conv2d(store, cfg, h, cfg.image_shape[2], 3, 3, 1, "final_conv"))


def _gen_sndcgan(store, cfg, z, y, is_training):
  """sndcgan.Generator.apply (sndcgan.py:42-79); its batch_norm calls pass use_sn = G.spectral_norm."""
  sn, b = cfg.g_sn, z.shape[0]
  sh, sw, colors = cfg.image_shape
  c2 = lambda s: -(-s // 2)
  sh2, sw2 = c2(sh), c2(sw)
  sh4, sw4 = c2(sh2), c2(sw2)
  sh8, sw8 = c2(sh4), c2(sw4)
  h = onets.linear(store, cfg, z, sh8 * sw8 * 512, "g_fc1")
  h = torch.relu(_bn(store, cfg, h, z, is_training, "g_bn1", sn)).reshape(b, sh8, sw8, 512)
  for i, (hw, co) in enumerate((((sh4, sw4), 256), ((sh2, sw2), 128), ((sh, sw), 64))):
    h = onets.deconv2d(store, cfg, h, (b,) + hw + (co,), 4, 4, 2, "g_dc%d" % (i + 2))
    h = torch.relu(_bn(store, cfg, h, z, is_training, "g_bn%d" % (i + 2), sn))
  h = onets.deconv2d(store, cfg, h, (b, sh, sw, colors), 3, 3, 1, "g_dc5")
  return (torch.tanh(h) + 1.0) / 2.0


def _gen_dcgan(store, cfg, z, y, is_training):
  """dcgan.Generator.apply (dcgan.py:39-84)."""
  sn, b = cfg.g_sn, z.shape[0]
  sh, sw, colors = cfg.image_shape
  c2 = lambda s: -(-s // 2)
  sizes = [(sh, sw)]
  for _ in range(4):
    sizes.append((c2(sizes[-1][0]), c2(sizes[-1][1])))
  h = onets.linear(store, cfg, z, 512 * sizes[4][0] * sizes[4][1], "g_fc1").reshape(-1, sizes[4][0], sizes[4][1], 512)
  h = torch.relu(_bn(store, cfg, h, z, is_training, "g_bn1", sn))
  for i, co in enumerate((256, 128, 64)):
    h = onets.deconv2d(store, cfg, h, (b,) + sizes[3 - i] + (co,), 5, 5, 2, "g_dc%d" % (i + 1))
    h = torch.relu(_bn(store, cfg, h, z, is_training, "g_bn%d" % (i + 2), sn))
  h = onets.deconv2d(store, cfg, h, (b, sh, sw, colors), 5, 5, 2, "g_dc4")
  return 0.5 * torch.tanh(h) + 0.5


def _gen_biggan(store, cfg, z, y, is_training):
  """resnet_biggan.Generator.apply (resnet_biggan.py:223-302): block i normalises with z chunk i (or the whole z)."""
  sn = cfg.g_sn
  mult = onets._BIGGAN_G[cfg.image_shape[0]]
  cin, cout = [cfg.ch * c for c in mult[:-1]], [cfg.ch * c for c in mult[1:]]
  nb = len(cin)
  if cfg.embed_y:                     # created as the reference creates it; a self-modulated BigGAN does not read y
    onets.linear(store, cfg, y, cfg.embed_y_dim, "embed_y", use_sn=False, use_bias=False)
  if cfg.hierarchical_z:
    chunks = torch.chunk(z, nb + 1, dim=1)
    z0, z_per_block = chunks[0], chunks[1:]
  else:
    z0, z_per_block = z, nb * [z]
  h = onets.linear(store, cfg, z0, cin[0] * 16, "fc_noise", use_sn=sn).reshape(-1, 4, 4, cin[0])
  attn = set(cfg.g_attention.split(","))
  for i in range(nb):
    name = "B%d" % (i + 1)
    h = _biggan_block(store, cfg, h, name, cin[i], cout[i], z_per_block[i], is_training, sn)
    if name in attn:
      h = onets.non_local_block(store, cfg, h, "non_local_block", sn)
  h = torch.relu(onets.batch_norm(store, cfg, h, is_training, name="final_norm"))
  h = onets.conv2d(store, cfg, h, cfg.image_shape[2], 3, 3, 1, "final_conv", use_sn=sn)
  return (torch.tanh(h) + 1.0) / 2.0


def _gen_biggan_deep(store, cfg, z, y, is_training):
  """resnet_biggan_deep.Generator.apply (resnet_biggan_deep.py:243-311): every block normalises with [z, embed(y)]."""
  sn = cfg.g_sn
  mult = onets._DEEP_G[cfg.image_shape[0]]
  cin, cout = [cfg.ch * c for c in mult[:-1]], [cfg.ch * c for c in mult[1:]]
  if cfg.embed_y:
    y = onets.linear(store, cfg, y, cfg.embed_y_dim, "embed_y", use_sn=False, use_bias=False)
  if y is not None:
    z = torch.cat([z, y], dim=1)
  h = onets.linear(store, cfg, z, cin[0] * 16, "fc_noise", use_sn=sn).reshape(-1, 4, 4, cin[0])
  for i in range(len(cin)):
    scale = "none" if i % 2 == 0 else "up"
    h = _biggan_deep_block(store, cfg, h, "B%d" % (i + 1), cin[i], cout[i], scale, z, is_training, sn)
    if scale == "up" and h.shape[1] == 64:
      h = onets.non_local_block(store, cfg, h, "non_local_block", sn)
  h = torch.relu(onets.batch_norm(store, cfg, h, is_training, name="final_norm"))
  h = onets.conv2d(store, cfg, h, cfg.image_shape[2], 3, 3, 1, "final_conv", use_sn=sn)
  return (torch.tanh(h) + 1.0) / 2.0


GENERATORS = {"resnet_cifar_arch": _gen_resnet_cifar, "resnet5_arch": _gen_resnet5, "sndcgan_arch": _gen_sndcgan,
              "dcgan_arch": _gen_dcgan, "resnet_biggan_arch": _gen_biggan, "resnet_biggan_deep_arch": _gen_biggan_deep}


@contextlib.contextmanager
def self_modulated_generators():
  """Inside this scope the generator of an oracle whose Cfg has `self_modulated = True` normalises with
  self_modulated_batch_norm (its discriminator and BigGAN's plain final_norm are untouched)."""
  saved = dict(onets._GENS)

  def dispatch(arch):
    def gen(store, cfg, z, y, is_training):
      fn = GENERATORS[arch] if getattr(cfg, "self_modulated", False) else saved[arch]
      return fn(store, cfg, z, y, is_training)
    return gen
  onets._GENS.update({arch: dispatch(arch) for arch in GENERATORS})
  try:
    yield
  finally:
    onets._GENS.clear()
    onets._GENS.update(saved)
