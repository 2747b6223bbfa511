"""TEST INFRASTRUCTURE ONLY: the DRAGAN and L2 penalties (reference penalty_lib.py:33-57, 85-103) on the oracle side.

`dragan_penalty` and `l2_penalty` restate the reference op by op on PyTorch-CPU, in the oracle's dtype (so the float64
twin is float64 throughout, moments included).  DRAGAN's uniform draw is fed, [B, H, W, C], through the oracle's
`alphas` argument; tests regenerate it from the device stream at the seed and step the engine used (`uniform`).
`penalties()` adds both as branches of oracle.gan.get_penalty_loss, leaving its own branches as they are."""
import contextlib

import numpy as np
import torch

from oracle import gan as ogan
from oracle import nets as onets


def dragan_penalty(store, cfg, x, y, is_training, u):
  """penalty_lib.py:46-56: tf.nn.moments over every axis (variance of x - stop_gradient(mean)), std = sqrt(var),
  x_noisy = clip(x + std * (u - 0.5), 0, 1), then WGAN-GP's slope penalty at x_noisy."""
  mean = x.mean()
  var = torch.square(x - mean).mean()
  noisy = torch.clamp(x + torch.sqrt(var) * (u - 0.5), 0.0, 1.0).detach().requires_grad_(True)
  logits = onets.discriminator(store, cfg, noisy, y, is_training)[1]
  g = torch.autograd.grad(logits.sum(), noisy, create_graph=True)[0]
  slopes = torch.sqrt(0.0001 + (g * g).sum(dim=(1, 2, 3)))
  return ((slopes - 1.0) ** 2).mean()


def kernel_names(store):
  """The discriminator's trainable `.../kernel` variables (the reference's `/kernel:0` suffix), rotation head included."""
  return [k for k in store.trainable if k.split("/")[0].startswith("discriminator") and k.endswith("/kernel")]


def l2_penalty(store):
  """penalty_lib.py:98-102: reduce_mean([tf.nn.l2_loss(w) for w in the kernels])."""
  return torch.stack([torch.square(store.vars[k]).sum() / 2 for k in kernel_names(store)]).mean()


@contextlib.contextmanager
def penalties():
  """Inside this scope oracle.gan.get_penalty_loss also knows "dragan_penalty" (the fed `alpha` is the uniform draw) and
  "l2_penalty"."""
  base = ogan.get_penalty_loss

  def get_penalty_loss(fn, store, cfg, x, x_fake, y, is_training, alpha=None):
    if fn == "dragan_penalty":
      return dragan_penalty(store, cfg, x, y, is_training, alpha)
    if fn == "l2_penalty":
      return l2_penalty(store)
    return base(fn, store, cfg, x, x_fake, y, is_training, alpha)
  ogan.get_penalty_loss = get_penalty_loss
  try:
    yield
  finally:
    ogan.get_penalty_loss = base


def uniform(seed, offset, n):
  """Elements offset .. offset + n - 1 of the counter-based stream (cgan_random_uniform): SplitMix64 of (seed, i + 1),
  the top 24 bits over 2^24."""
  with np.errstate(over="ignore"):
    z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * (np.uint64(offset) + np.arange(1, n + 1, dtype=np.uint64))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
  return (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def batch_std(x):
  """sqrtf of the float64 variance of all of x rounded once to fp32: the std the device entry uses."""
  x64 = np.asarray(x, np.float64)
  return np.sqrt(np.float32(((x64 - x64.mean()) ** 2).mean()))


def perturb(x, u, std):
  """The device entry's elementwise pass given u and std: clip(x + std * (u - 0.5), 0, 1), every operation in fp32."""
  x = np.asarray(x, np.float32)
  y = x + np.float32(std) * (np.asarray(u, np.float32).reshape(x.shape) - np.float32(0.5))
  return np.minimum(np.maximum(y, np.float32(0)), np.float32(1)).astype(np.float32)
