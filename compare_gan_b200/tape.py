"""Host-side tape for reverse-mode differentiation over the C-ABI kernels.

TensorFlow's graph autodiff (tf.gradients, used by optimizer.minimize at
gans/modular_gan.py:478-497 and by the gradient penalties at gans/penalty_lib.py:78) is
replaced by a small tape: every op in `kernels.py` launches sm_90a kernels through the C-ABI
and records a vector-Jacobian closure that is itself written in terms of those ops, so the
WGAN-GP second backward needs no special casing.  PyTorch is used for device memory only
(`torch.empty`); no torch op, no torch.autograd, on this path.  The Python overhead disappears
when the whole cycle is captured into a CUDA graph (gans/modular_gan.py of this package).
"""
import contextlib
import weakref

import torch


class DT(object):
  """Device tensor: float32 (or int32 labels), C-contiguous; 4-D tensors are NHWC."""
  __slots__ = ("t", "node", "req", "tf32", "relu_of", "premasked_for", "tan", "__weakref__")

  def __init__(self, t, req=False):
    assert t.is_contiguous()
    self.t = t
    self.node = None
    self.req = req
    # True when a kernel stored this tensor rounded to the nearest TF32 value (math_mode 1): tensor-core contractions
    # that read it skip their operand-rounding pass (include/cgan_b200.h, CGAN_CONV_IN_TF32)
    self.tf32 = False
    # fusion of a (leaky-)ReLU backward into the epilogue of the contraction that produces its incoming gradient:
    # relu_of = (ref, leak) marks this tensor as the output of a (leaky-)ReLU whose gradient mask is sign(ref);
    # premasked_for = id(tensor) marks a gradient that already carries that tensor's mask (kernels.conv2d_dgrad)
    self.relu_of = None
    self.premasked_for = None
    # forward mode (metrics/jacobian_conditioning.py): a DT [shape[0] * k, ...] holding k tangents of every sample of this
    # tensor, sample-major (row block b * k + j is tangent j of sample b); None when this tensor carries no tangent
    self.tan = None

  @property
  def shape(self):
    return tuple(self.t.shape)

  @property
  def ptr(self):
    return self.t.data_ptr()

  @property
  def numel(self):
    return self.t.numel()

  def view(self, *shape):
    """Zero-copy reshape WITHOUT a tape link (use kernels.reshape inside differentiated code)."""
    v = DT(self.t.view(*shape))
    v.tf32 = self.tf32
    return v

  def cpu(self):
    return self.t.detach().cpu().numpy()


class Node(object):
  """`out` is held weakly: DT -> node -> inputs is then a DAG without reference cycles, so dropping the loss tensor
  frees a whole sub-step's activation stash immediately by reference counting (a cyclic-GC delay here costs tens of GB)."""
  __slots__ = ("name", "inputs", "vjp", "_out")

  def __init__(self, name, inputs, vjp, out):
    self.name, self.inputs, self.vjp, self._out = name, inputs, vjp, weakref.ref(out)

  @property
  def out(self):
    return self._out()


_RECORD = [True]


@contextlib.contextmanager
def no_record():
  _RECORD.append(False)
  try:
    yield
  finally:
    _RECORD.pop()


@contextlib.contextmanager
def record(flag=True):
  _RECORD.append(flag)
  try:
    yield
  finally:
    _RECORD.pop()


def recording():
  return _RECORD[-1]


def attach(name, out, inputs, vjp):
  """Record `out = op(inputs)`; vjp(gout, needs) -> list of grads (None where not needed).  An op that has a forward-mode
  rule sets out.tan before it attaches; one that does not must never drop an input's tangent silently."""
  if out.tan is None and any(i is not None and i.tan is not None for i in inputs):
    raise NotImplementedError("forward-mode tangents through %s are not implemented" % name)
  if _RECORD[-1] and any(i is not None and i.req for i in inputs):
    out.req = True
    out.node = Node(name, inputs, vjp, out)
  return out


def _topo(roots):
  order, seen = [], set()
  stack = [(r, False) for r in roots if r.node is not None]
  while stack:
    t, done = stack.pop()
    if done:
      order.append(t.node)
      continue
    if id(t) in seen:
      continue
    seen.add(id(t))
    stack.append((t, True))
    for i in t.node.inputs:
      if i is not None and i.node is not None and id(i) not in seen:
        stack.append((i, False))
  return order   # inputs before consumers


_ADD_TAKES_TENSOR = {}
_SINKS = [None]
_CONSUMERS = [None]


def sole_consumer(t):
  """True while a backward pass runs and exactly one differentiated op consumed `t` (its gradient has one contribution)."""
  d = _CONSUMERS[-1]
  return d is not None and d.get(id(t), 0) == 1


def take_sink(t):
  """During backward(..., sinks=...): the caller-provided destination for the gradient of leaf `t` (a view into a flat
  gradient buffer), handed out ONCE — to the first vjp that produces a contribution for `t`, which then writes it there
  instead of into fresh memory.  Later contributions are accumulated by add_fn as usual."""
  d = _SINKS[-1]
  if d is None or t is None:
    return None
  return d.pop(id(t), None)


def grad_accumulator(fn):
  """Marks `fn(prev, g, tensor)` as an accumulation function that wants to know which tensor the gradient is for."""
  _ADD_TAKES_TENSOR[fn] = True
  return fn


def backward(roots, wrt, add_fn, create_graph=False, sinks=None):
  """roots: list of (DT, seed) with seed a DT or None (meaning d(root)/d(root)=1 for scalar-loss ops).
  Returns the list of gradients for `wrt` (None where unreachable).  `sinks` ({id(leaf): DT}) offers destinations for
  leaf gradients (see take_sink); a returned gradient may therefore alias its sink."""
  order = _topo([r for r, _ in roots])
  dep = set(id(w) for w in wrt)
  outs = {}                      # strong refs for the duration of this backward pass
  for node in order:
    out = node.out
    if out is None:
      continue
    outs[id(node)] = out
    if any(i is not None and id(i) in dep for i in node.inputs):
      dep.add(id(out))
  grads = {}
  keep = set(id(w) for w in wrt)
  for r, seed in roots:
    if id(r) in dep:
      grads[id(r)] = ("seed", seed) if id(r) not in grads else grads[id(r)]
  _SINKS.append(dict(sinks) if sinks else None)
  ncons = {}
  for node in order:
    if id(node) in outs and id(outs[id(node)]) in dep:
      for i in node.inputs:
        if i is not None and id(i) in dep:
          ncons[id(i)] = ncons.get(id(i), 0) + 1
  _CONSUMERS.append(None if create_graph else ncons)
  try:
   with record(create_graph):
    for node in reversed(order):
      if id(node) not in outs:
        continue
      oid = id(outs[id(node)])
      if oid not in grads or oid not in dep:
        continue
      g = grads[oid]
      if isinstance(g, tuple):
        g = g[1]
      needs = [i is not None and id(i) in dep for i in node.inputs]
      if not any(needs):
        continue
      gins = node.vjp(g, needs)
      for i, gi in zip(node.inputs, gins):
        if gi is None or i is None or id(i) not in dep:
          continue
        if id(i) in grads:
          prev = grads[id(i)]
          grads[id(i)] = add_fn(prev, gi, i) if _ADD_TAKES_TENSOR.get(add_fn) else add_fn(prev, gi)
        else:
          grads[id(i)] = gi
      if oid not in keep:
        del grads[oid]
  finally:
    _SINKS.pop()
    _CONSUMERS.pop()
  out = []
  for w in wrt:
    g = grads.get(id(w))
    out.append(None if g is None or isinstance(g, tuple) else g)
  return out
