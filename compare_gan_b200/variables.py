"""tf.get_variable / tf.variable_scope stand-in over device memory.

Variable names reproduce the reference's checkpoint key space (e.g. generator/B1/up_conv1/kernel,
.../kernel/u_var, .../bn1/moving_mean, .../bn1/accu/accu_mean; pinned by
architectures/resnet_norm_test.py).  Trainable variables of each network are packed into ONE flat
float32 buffer (and one flat gradient / Adam-m / Adam-v buffer) so the optimizer is a single fused
kernel and the data-parallel exchange is a single NCCL all-reduce (CrossShardOptimizer,
gans/modular_gan.py:606-616).
"""
import contextlib
from collections import OrderedDict

import numpy as np
import torch

from . import kernels as K
from .tape import DT

ALIGN = 64   # floats (256 B): keeps every packed variable 16B-aligned for vector loads / TMA


class VariableStore(object):

  def __init__(self, seed=0):
    self.vars = OrderedDict()        # name -> DT
    self.trainable = OrderedDict()   # name -> DT (subset)
    self.init_values = OrderedDict() # name -> numpy initial value (host)
    self._scope = []
    self.rng = np.random.RandomState(seed)
    self.flat = {}                   # prefix -> dict(param=DT, grad=DT, views=OrderedDict name -> (off, n))

  # ---- scopes ---------------------------------------------------------------------------
  @contextlib.contextmanager
  def scope(self, name):
    self._scope.append(name)
    try:
      yield
    finally:
      self._scope.pop()

  @contextlib.contextmanager
  def at_scope(self, scope):
    """Runs the body in the scope path `scope` (a list of names), whatever scope is open."""
    saved, self._scope = self._scope, list(scope)
    try:
      yield
    finally:
      self._scope = saved

  def full_name(self, name):
    return "/".join(self._scope + [name])

  # ---- creation ---------------------------------------------------------------------------
  def get(self, name, shape, initializer, trainable=True):
    """tf.get_variable with reuse=AUTO_REUSE; `initializer(rng, shape) -> np.float32 array`."""
    full = self.full_name(name)
    shape = tuple(int(s) for s in shape)
    if full in self.vars:
      v = self.vars[full]
      if v.shape != shape:
        raise ValueError("Trying to share variable %s, but specified shape %s and found shape %s." %
                         (full, shape, v.shape))
      return v
    a = np.asarray(initializer(self.rng, shape), np.float32).reshape(shape)
    v = K.from_numpy(a, req=trainable)
    self.vars[full] = v
    self.init_values[full] = a
    if trainable:
      self.trainable[full] = v
    return v

  def trainable_under(self, prefix):
    """Trainable variables of a network.  The reference selects them by substring (`self._name in var.name`,
    architectures/abstract_arch.py:43-45), which is how SSGAN's `discriminator_rotation/...` head trains with the
    discriminator: here the top-level scope must START with the network's name."""
    return OrderedDict((k, v) for k, v in self.trainable.items() if k.split("/")[0].startswith(prefix))

  # ---- flat packing -----------------------------------------------------------------------
  def pack(self, prefix):
    """Move the trainable variables under `prefix/` into one flat buffer (views keep their DT identity)."""
    tv = self.trainable_under(prefix)
    off, views = 0, OrderedDict()
    for k, v in tv.items():
      views[k] = (off, v.numel)
      off += (v.numel + ALIGN - 1) // ALIGN * ALIGN
    total = max(off, ALIGN)
    dev = K._RT["device"]
    param = torch.zeros(total, dtype=torch.float32, device=dev)
    grad = torch.zeros(total, dtype=torch.float32, device=dev)
    for k, v in tv.items():
      o, n = views[k]
      param[o:o + n].copy_(v.t.reshape(-1))
      v.t = param[o:o + n].view(v.shape)
    self.flat[prefix] = {"param": DT(param), "grad": DT(grad), "views": views, "total": total}
    return self.flat[prefix]

  def grad_view(self, prefix, name):
    f = self.flat[prefix]
    o, n = f["views"][name]
    return DT(f["grad"].t[o:o + n])

  # ---- host I/O (checkpoint key space) ------------------------------------------------------
  def state_numpy(self):
    return OrderedDict((k, v.cpu().copy()) for k, v in self.vars.items())

  def load_numpy(self, state, strict=False):
    for k, a in state.items():
      if k not in self.vars:
        if strict:
          raise KeyError(k)
        continue
      v = self.vars[k]
      v.t.copy_(torch.from_numpy(np.asarray(a, np.float32).reshape(v.shape)).to(v.t.device))

  def reset_to_init(self):
    self.load_numpy(self.init_values)


_CURRENT = [None]


def current():
  if _CURRENT[0] is None:
    raise RuntimeError("no active VariableStore: wrap model code in `with variables.use(store):`")
  return _CURRENT[0]


@contextlib.contextmanager
def use(store):
  prev = _CURRENT[0]
  _CURRENT[0] = store
  try:
    yield store
  finally:
    _CURRENT[0] = prev


def variable_scope(name):
  return current().scope(name)


def get_variable(name, shape, initializer, trainable=True):
  return current().get(name, shape, initializer, trainable)
