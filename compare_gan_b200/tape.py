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
  __slots__ = ("name", "inputs", "vjp", "_out", "chain")

  def __init__(self, name, inputs, vjp, out):
    self.name, self.inputs, self.vjp, self._out = name, inputs, vjp, weakref.ref(out)
    # a segment's node (see segment): the names of the ops its replay will record along the first inputs, for producers()
    self.chain = None

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
  p = _PASS[-1]
  if p is not None and not p.replay:
    p.saw(name, out, inputs)
  if _RECORD[-1] and any(i is not None and i.req for i in inputs):
    out.req = True
    out.node = Node(name, inputs, vjp, out)
  return out


def producers(t, n):
  """Names of the ops that produced `t`, its first input, that input's first input, ... (at most n, fewer where the chain
  reaches a tensor without a node).  A segment's output answers with the chain its replay records."""
  names = []
  while len(names) < n and t is not None and t.node is not None:
    if t.node.chain is not None:
      return (names + list(t.node.chain))[:n]
    names.append(t.node.name)
    t = t.node.inputs[0]
  return names


def _topo(roots, stop=()):
  """Nodes reachable from `roots`, inputs before consumers; tensors in `stop` (ids) are not expanded."""
  order, seen = [], set(stop)
  stack = [(r, False) for r in roots if r.node is not None and id(r) not in seen]
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
_GRADS = [None]      # (gradient dict, add_fn) of the running backward pass


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
  return _backward(roots, wrt, add_fn, create_graph, dict(sinks) if sinks else None)


def _backward(roots, wrt, add_fn, create_graph, sinks, stop=(), grads=None, consumers=None):
  """backward() over the sub-graph above `stop` (ids of tensors not expanded).  `grads` ({id: partial gradient}) carries
  the sums a caller has accumulated so far, `consumers` ({id: count}) the consumers a tensor has outside the sub-graph;
  `sinks` is the sink dict itself (shared with the caller, not copied)."""
  order = _topo([r for r, _ in roots], stop)
  dep = set(id(w) for w in wrt)
  outs = {}                      # strong refs for the duration of this backward pass
  for node in order:
    out = node.out
    if out is None:
      continue
    outs[id(node)] = out
    if any(i is not None and id(i) in dep for i in node.inputs):
      dep.add(id(out))
  grads = {} if grads is None else grads
  keep = set(id(w) for w in wrt)
  for r, seed in roots:
    if id(r) in dep:
      grads[id(r)] = ("seed", seed) if id(r) not in grads else grads[id(r)]
  _SINKS.append(sinks)
  ncons = {}
  for node in order:
    if id(node) in outs and id(outs[id(node)]) in dep:
      for i in node.inputs:
        if i is not None and id(i) in dep:
          ncons[id(i)] = ncons.get(id(i), 0) + 1
  for k, v in (consumers or {}).items():
    if k in ncons:
      ncons[k] += v
  _CONSUMERS.append(None if create_graph else ncons)
  _GRADS.append((grads, add_fn))
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
    _GRADS.pop()
  out = []
  for w in wrt:
    g = grads.get(id(w))
    out.append(None if g is None or isinstance(g, tuple) else g)
  return out


# ------------------------------------------------------------------------------------ recomputed segments
# A segment trades its activation stash for one more forward: the first pass runs with recording off and attaches ONE node
# holding only the segment's inputs and the trainable leaves it read; that node's vjp replays the forward with recording
# on and runs an inner backward over the replayed sub-graph.  The replay must reproduce the first pass bit for bit and
# cause no second side effect, so an op with state (batch-norm moments and moving averages, the spectral-norm power
# iteration) computes through replayed(), which records its result in the first pass and serves it back, in call order,
# during the replay; observers stay silent while replaying().

_SEGMENTS = [False]  # whether segment() cuts segments in the running network call
_PASS = [None]       # the segment pass in progress


class _Pass(object):
  __slots__ = ("replay", "log", "pos", "leaves", "_seen", "_chains")

  def __init__(self, replay, log):
    self.replay, self.log, self.pos = replay, log, 0
    self.leaves, self._seen, self._chains = [], set(), {}

  def saw(self, name, out, inputs):
    """attach() during a first pass: collect the trainable leaves, and the producer chain of `out`."""
    for i in inputs:
      if i is not None and i.req and i.node is None and id(i) not in self._seen:
        self._seen.add(id(i))
        self.leaves.append(i)
    self._chains[id(out)] = (weakref.ref(out), ((name,) + self.chain(inputs[0] if inputs else None))[:4])

  def chain(self, t):
    if t is None:
      return ()
    hit = self._chains.get(id(t))
    if hit is not None and hit[0]() is t:      # (an id is only trusted while its tensor is alive)
      return hit[1]
    return tuple(producers(t, 4))


@contextlib.contextmanager
def segments(flag):
  """segment() cuts segments inside this scope only when `flag` is true (a network's recompute decision)."""
  _SEGMENTS.append(bool(flag))
  try:
    yield
  finally:
    _SEGMENTS.pop()


def replaying():
  return _PASS[-1] is not None and _PASS[-1].replay


def replayed(compute):
  """compute() for an op with side effects: its result is recorded in a segment's first pass and served back, without
  calling compute, when the segment is replayed."""
  p = _PASS[-1]
  if p is None:
    return compute()
  if p.replay:
    p.pos += 1
    return p.log[p.pos - 1]
  v = compute()
  p.log.append(v)
  return v


def segment(fn, inputs):
  """out = fn(*inputs) as a recomputed segment (see above).  `inputs` lists the segment's tensor inputs (None allowed),
  the activation it continues first.  Outside segments(True), while not recording, or inside another segment's pass,
  this is fn(*inputs)."""
  if not (_SEGMENTS[-1] and _RECORD[-1]) or _PASS[-1] is not None:
    return fn(*inputs)
  first = _Pass(False, [])
  _PASS.append(first)
  try:
    with record(False):
      out = fn(*inputs)
  finally:
    _PASS.pop()
  if out.node is not None:
    return out                     # fn returned a recorded tensor (one of its inputs) unchanged: nothing to recompute
  ins = []
  for i in inputs:
    if i is not None and all(i is not j for j in ins):
      ins.append(i)
  leaves = [l for l in first.leaves if all(l is not j for j in ins)]
  # the continued activation goes last: the backward's walk then reaches the network before the segment's side inputs, as
  # it does through the block's own shortcut, and the partial sums of shared inputs grow in the stash path's order
  node_inputs = ins[1:] + leaves + ins[:1]
  stop = set(id(i) for i in ins)
  log, out_id, chain = first.log, id(out), first.chain(out)
  del first

  def vjp(g, needs):
    if _RECORD[-1]:
      raise NotImplementedError("second-order differentiation through a recomputed segment is not implemented")
    outer, add_fn = _GRADS[-1]
    ocons = _CONSUMERS[-1] or {}
    wrt = [i for i, n in zip(node_inputs, needs) if n]
    p = _Pass(True, log)
    _PASS.append(p)
    try:
      with record(True):
        out2 = fn(*inputs)
    finally:
      _PASS.pop()
    if p.pos != len(log):
      raise RuntimeError("a segment's replay consumed %d of the %d recorded results" % (p.pos, len(log)))
    seed = g
    if getattr(g, "premasked_for", None) == out_id:       # a consumer applied the output's ReLU mask: tell the replay's op
      seed = DT(g.t)
      seed.tf32, seed.premasked_for = g.tf32, id(out2)
    # the inner pass continues the caller's partial sums, hands leaf gradients to the caller's sinks, and counts the
    # consumers each input has outside the segment; its results replace the caller's partial sums
    grads = _backward([(out2, seed)], wrt, add_fn, False, _SINKS[-1], stop=stop,
                      grads={id(w): outer[id(w)] for w in wrt if id(w) in outer},
                      consumers={id(i): ocons.get(id(i), 1) - 1 for i in ins})
    del out2                       # the replayed stash goes here
    for w, gw in zip(wrt, grads):
      if gw is not None:
        outer[id(w)] = gw
    return [None] * len(node_inputs)

  attach("segment", out, node_inputs, vjp)
  if out.node is not None:
    out.node.chain = chain
  return out
