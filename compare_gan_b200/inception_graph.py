"""Importer for TF-GAN's frozen Inception graph: `inceptionv1_for_inception_score.pb`, alone or inside
`frozen_inception_v1_2015_12_05.tar.gz` (the file the reference downloads, eval_utils.py:41-49, and reads `pool_3:0` /
`logits:0` from, eval_utils.py:165-175), turned into the weight dict `inception.InceptionV3` takes.

The GraphDef is decoded with `tf_checkpoint`'s protobuf wire-format helpers.  The import is structural: only the names
of TF-GAN's contract are relied on (the input `Mul`, the outputs `pool_3` and `logits`); every other node is identified
by its op and its position.  The walk goes backwards from `pool_3` to `Mul` and interprets Conv2D -> batch norm
(inference constants) -> Relu chains, max / average pools and (nested, flattened) channel concats, passing through
Identity and CheckNumerics.  The interpreted network must be `inception.SPEC` in order (kernel shapes, strides, paddings,
pool kinds and sizes, concat branch order), followed by `pool_3` -> (Reshape / Squeeze) -> MatMul -> BiasAdd / Add ->
`logits` with a 2048 -> 1008 layer.  Anything else raises ValueError naming the node, its op and what SPEC expected;
branches are never permuted.  Batch norm is folded into the convolution in float64: s = gamma / sqrt(var + eps)
(gamma = 1 without scale_after_normalization), kernel = fp32(W * s), bias = fp32(beta - mean * s).

    python -m compare_gan_b200.inception_graph SRC OUT.npz     # SRC: the .pb or the tarball; then CGAN_INCEPTION_NPZ=OUT.npz
"""
import os
import struct
import sys
import tarfile

import numpy as np

from . import inception
from .tf_checkpoint import DTYPES, _parse_message, _read_varint, _signed64

GRAPH_MEMBER = "inceptionv1_for_inception_score.pb"
INPUT, POOL, LOGITS = "Mul", "pool_3", "logits"
FINAL_HW = 8          # the map SPEC leaves at 299x299, which pool_3 averages
_PASS = ("Identity", "CheckNumerics")
_BN = ("BatchNormWithGlobalNormalization", "FusedBatchNorm", "FusedBatchNormV2", "FusedBatchNormV3")
_CONCAT = ("Concat", "ConcatV2")
_KNOWN = set(_PASS + _BN + _CONCAT + ("Conv2D", "Relu", "MaxPool", "AvgPool", "Const", "Reshape", "Squeeze", "MatMul",
                                     "BiasAdd", "Add"))


# ---- GraphDef decoding -----------------------------------------------------------------------------------------------

def _f32(bits):
  return struct.unpack("<f", struct.pack("<I", bits))[0]


def _floats(values):
  """A repeated float field, packed (one length-delimited run) or not (fixed32 entries)."""
  out = []
  for v in values:
    out.extend(np.frombuffer(v, "<f4").tolist() if isinstance(v, bytes) else [_f32(v)])
  return out


def _ints(values):
  """A repeated varint field, packed or not."""
  out = []
  for v in values:
    if isinstance(v, bytes):
      pos = 0
      while pos < len(v):
        x, pos = _read_varint(v, pos)
        out.append(_signed64(x))
    else:
      out.append(_signed64(v))
  return out


def _tensor(buf, where):
  """TensorProto: dtype 1, tensor_shape 2 (dim 2 {size 1}), tensor_content 4, float_val 5, int_val 7.  Fewer values
  than the shape holds repeat the last one (none: zeros), as TensorFlow fills them."""
  f = _parse_message(buf)
  code = f.get(1, [0])[0]
  if code not in DTYPES:
    raise ValueError("%s: tensor dtype %d is not supported" % (where, code))
  dt = np.dtype(DTYPES[code])
  dims = _parse_message(f[2][0]).get(2, []) if 2 in f else []
  shape = tuple(_signed64(_parse_message(d).get(1, [0])[0]) for d in dims)
  n = int(np.prod(shape, dtype=np.int64))
  if 4 in f:
    a = np.frombuffer(f[4][0], dt.newbyteorder("<"))
  elif code == 1:
    a = np.array(_floats(f.get(5, [])), dt)
  elif dt.kind == "i":
    a = np.array(_ints(f.get(7, [])), dt)
  else:
    raise ValueError("%s: %s tensor without tensor_content is not supported" % (where, dt))
  if 4 not in f and a.size < n:
    a = np.concatenate([a, np.full(n - a.size, a[-1] if a.size else 0, dt)])
  if a.size != n:
    raise ValueError("%s: %d values for tensor shape %s" % (where, a.size, shape))
  return a.astype(dt).reshape(shape)


def _attr(buf):
  """AttrValue: list 1 (ListValue: s 2, i 3, f 4), s 2, i 3, f 4, b 5; a tensor 8 is kept encoded until it is used."""
  f = _parse_message(buf)
  if 1 in f:
    lv = _parse_message(f[1][0])
    return _ints(lv.get(3, [])) or _floats(lv.get(4, [])) or [s.decode() for s in lv.get(2, [])]
  if 2 in f:
    return f[2][0].decode()
  if 3 in f:
    return _signed64(f[3][0])
  if 4 in f:
    return _f32(f[4][0])
  if 5 in f:
    return bool(f[5][0])
  if 8 in f:
    return f[8][0]
  return None


class Node(object):
  """NodeDef: name 1, op 2, input 3 (control inputs `^name` dropped, `name:k` kept as (name, k)), attr 5."""

  def __init__(self, buf):
    f = _parse_message(buf)
    self.name = f[1][0].decode()
    self.op = f.get(2, [b""])[0].decode()
    self.inputs = []
    for s in f.get(3, []):
      s = s.decode()
      if not s.startswith("^"):
        name, _, k = s.partition(":")
        self.inputs.append((name, int(k) if k else 0))
    self.attr = {}
    for entry in f.get(5, []):
      e = _parse_message(entry)
      self.attr[e[1][0].decode()] = _attr(e.get(2, [b""])[0])

  def __repr__(self):
    return "node %r (op %s)" % (self.name, self.op)


def parse_graph(data):
  """{name: Node} of a serialized GraphDef (node = field 1)."""
  nodes = {}
  for buf in _parse_message(data).get(1, []):
    node = Node(buf)
    nodes[node.name] = node
  return nodes


def read_graph_bytes(path):
  """The GraphDef bytes of `path`: the .pb itself, or the `inceptionv1_for_inception_score.pb` member of a tarball."""
  if tarfile.is_tarfile(path):
    with tarfile.open(path) as tar:
      for m in tar.getmembers():
        if m.isfile() and os.path.basename(m.name) == GRAPH_MEMBER:
          return tar.extractfile(m).read()
    raise ValueError("%s: the archive has no member named %s" % (path, GRAPH_MEMBER))
  with open(path, "rb") as f:
    return f.read()


# ---- structural import -----------------------------------------------------------------------------------------------

def _paths(items):
  """The concat-free paths of a SPEC branch: a trailing split fans out into one path per sub-branch, as a flattened
  concat lists them."""
  if items and items[-1][0] == "split":
    return [items[:-1] + p for br in items[-1][1] for p in _paths(br)]
  return [items]


class _Importer(object):

  def __init__(self, nodes):
    self.nodes = nodes
    self.shapes = {name: (kh, kw, cin, cout) for name, kh, kw, cin, cout in inception.walk_convs()}
    self.conv_of = {}        # SPEC conv name -> the Relu node that computes it
    self.weights = {}

  def node(self, name):
    if name not in self.nodes:
      raise ValueError("the graph has no node named %r" % name)
    return self.nodes[name]

  def follow(self, node, i=0):
    """The node feeding data input i of `node`, through Identity / CheckNumerics."""
    while True:
      if i >= len(node.inputs):
        raise ValueError("%r has %d data inputs, input %d expected" % (node, len(node.inputs), i))
      name, k = node.inputs[i]
      src = self.node(name)
      if k != 0:
        raise ValueError("%r reads output %d of %r; only output 0 is interpreted" % (node, k, src))
      if src.op not in _PASS:
        return src
      node, i = src, 0

  @staticmethod
  def expect(node, ok, what):
    if not ok:
      unknown = "" if node.op in _KNOWN else " (an op the importer does not interpret)"
      raise ValueError("%r%s: SPEC expects %s" % (node, unknown, what))

  def const(self, node, i, shape, what):
    src = self.follow(node, i)
    self.expect(src, src.op == "Const", "a constant %s of shape %s as input %d of %r" % (what, shape, i, node))
    value = src.attr.get("value")
    self.expect(src, isinstance(value, bytes), "a tensor value for %s" % what)
    a = _tensor(value, src.name)
    if shape is not None and a.shape != tuple(shape):
      raise ValueError("%r: %s has shape %s, SPEC expects %s" % (src, what, a.shape, tuple(shape)))
    return a

  def nhwc(self, node, what):
    fmt = node.attr.get("data_format", "NHWC")
    self.expect(node, fmt == "NHWC", "data_format NHWC for %s, not %s" % (what, fmt))

  def window(self, node, key, k, what):
    self.expect(node, node.attr.get(key) == [1, k, k, 1], "%s [1, %d, %d, 1] for %s, not %s"
                % (key, k, k, what, node.attr.get(key)))

  def conv(self, relu, full, stride, padding):
    """Relu <- batch norm <- Conv2D computing SPEC's conv `full`; folds the BN and returns the Conv2D's input node."""
    what = "convolution %s" % full
    if full in self.conv_of:
      self.expect(relu, relu is self.conv_of[full], "the node %r computing %s in every branch that shares it"
                  % (self.conv_of[full].name, full))
      return self.follow(self.follow(self.follow(relu)))
    self.expect(relu, relu.op == "Relu", "Relu ending %s" % what)
    bn = self.follow(relu)
    self.expect(bn, bn.op in _BN, "batch norm (%s) of %s" % (" / ".join(_BN), what))
    conv = self.follow(bn)
    self.expect(conv, conv.op == "Conv2D", "Conv2D of %s" % what)
    self.nhwc(conv, what)
    self.window(conv, "strides", stride, what)
    self.expect(conv, conv.attr.get("padding") == padding, "padding %s for %s, not %s"
                % (padding, what, conv.attr.get("padding")))
    self.expect(conv, conv.attr.get("dilations", [1, 1, 1, 1]) == [1, 1, 1, 1], "no dilation for %s" % what)
    kh, kw, cin, cout = self.shapes[full]
    w = self.const(conv, 1, (kh, kw, cin, cout), "the kernel of %s" % full)
    if bn.op == "BatchNormWithGlobalNormalization":
      mean, var, beta, gamma = (self.const(bn, i, (cout,), "%s of %s" % (p, full)) for i, p in
                                enumerate(("mean", "variance", "beta", "gamma"), 1))
      for key in ("variance_epsilon", "scale_after_normalization"):
        self.expect(bn, key in bn.attr, "the attribute %s" % key)
      eps, scaled = bn.attr["variance_epsilon"], bn.attr["scale_after_normalization"]
    else:
      gamma, beta, mean, var = (self.const(bn, i, (cout,), "%s of %s" % (p, full)) for i, p in
                                enumerate(("scale", "offset", "mean", "variance"), 1))
      eps, scaled = bn.attr.get("epsilon", 1e-4), True
      self.expect(bn, bn.attr.get("is_training", True) is False, "is_training = false (inference batch norm)")
      self.nhwc(bn, what)
    f64 = np.float64
    s = (gamma.astype(f64) if scaled else 1.0) / np.sqrt(var.astype(f64) + f64(eps))
    self.weights["inception/%s/kernel" % full] = (w.astype(f64) * s).astype(np.float32)
    self.weights["inception/%s/bias" % full] = (beta.astype(f64) - mean.astype(f64) * s).astype(np.float32)
    self.conv_of[full] = relu
    return self.follow(conv)

  def pool(self, node, mode, k, s, padding):
    what = "the %s pool %dx%d / %d %s" % (mode, k, k, s, padding)
    self.expect(node, node.op == {"max": "MaxPool", "avg": "AvgPool"}[mode], what)
    self.nhwc(node, what)
    self.window(node, "ksize", k, what)
    self.window(node, "strides", s, what)
    self.expect(node, node.attr.get("padding") == padding, "padding %s for %s, not %s"
                % (padding, what, node.attr.get("padding")))
    return self.follow(node)

  def leaves(self, concat, what):
    """The tensors a channel concat joins, nested concats flattened in order."""
    self.expect(concat, concat.op in _CONCAT, "the channel concat of %s" % what)
    axis_at = 0 if concat.op == "Concat" else len(concat.inputs) - 1
    axis = self.const(concat, axis_at, None, "the concat axis")
    self.expect(concat, axis.size == 1 and int(axis.ravel()[0]) in (3, -1), "concatenation along channels (axis 3)")
    out = []
    for i in range(len(concat.inputs)):
      if i != axis_at:
        src = self.follow(concat, i)
        out.extend(self.leaves(src, what) if src.op in _CONCAT else [src])
    return out

  def seq(self, items, out, pre):
    """Matches SPEC `items` backwards from the node `out`; returns the node feeding the first item."""
    for it in reversed(items):
      if it[0] == "conv":
        _, name, _, _, _, stride, padding = it
        out = self.conv(out, pre + name, stride, padding)
      elif it[0] == "pool":
        out = self.pool(out, *it[1:])
      else:
        block = pre + it[1]
        paths = [p for br in it[2] for p in _paths(br)]
        leaves = self.leaves(out, "block " + block)
        self.expect(out, len(leaves) == len(paths), "%d concatenated branches for block %s, not %d"
                    % (len(paths), block, len(leaves)))
        starts = []
        for i, (path, leaf) in enumerate(zip(paths, leaves)):
          try:
            starts.append(self.seq(path, leaf, block + "/"))
          except ValueError as e:
            raise ValueError("branch %d of %r: %s" % (i, out, e))
        for i, s in enumerate(starts):
          self.expect(s, s is starts[0], "branch %d of %s to start from %r, as branch 0 does" % (i, block, starts[0]))
        out = starts[0]
    return out


def import_graph(nodes):
  """{`inception/<layer>/kernel|bias`: float32 array} of the parsed graph `nodes`, the dict InceptionV3 takes."""
  imp = _Importer(nodes)
  mul, pool = imp.node(INPUT), imp.node(POOL)
  imp.expect(pool, pool.op == "AvgPool", "pool_3 to average-pool the %dx%d map" % (FINAL_HW, FINAL_HW))
  imp.nhwc(pool, "pool_3")
  imp.window(pool, "ksize", FINAL_HW, "pool_3")
  imp.expect(pool, pool.attr.get("padding") == "VALID", "padding VALID for pool_3")
  start = imp.seq(inception.SPEC, imp.follow(pool), "")
  imp.expect(start, start is mul, "the network's first convolution to read the input %r" % INPUT)
  logits = imp.node(LOGITS)
  imp.expect(logits, logits.op in ("BiasAdd", "Add"), "BiasAdd / Add of the logits layer")
  mm_at = 0 if logits.op == "BiasAdd" or imp.follow(logits, 0).op == "MatMul" else 1
  mm = imp.follow(logits, mm_at)
  imp.expect(mm, mm.op == "MatMul", "MatMul of the logits layer")
  imp.expect(mm, not mm.attr.get("transpose_a", False), "transpose_a = false")
  x = imp.follow(mm, 0)
  while x.op in ("Reshape", "Squeeze"):
    x = imp.follow(x, 0)
  imp.expect(x, x is pool, "the logits layer to read %r" % POOL)
  head = (inception.NUM_CLASSES, inception.POOL_DIM) if mm.attr.get("transpose_b", False) else \
      (inception.POOL_DIM, inception.NUM_CLASSES)
  w = imp.const(mm, 1, None, "the logits weights")
  if w.shape != head:
    raise ValueError("%r: logits weights of shape %s (transpose_b = %s); SPEC expects a %d -> %d layer"
                     % (mm, w.shape, mm.attr.get("transpose_b", False), inception.POOL_DIM, inception.NUM_CLASSES))
  b = imp.const(logits, 1 - mm_at, (inception.NUM_CLASSES,), "the logits bias")
  imp.weights["inception/logits/kernel"] = np.ascontiguousarray(w.T if head[0] == inception.NUM_CLASSES else w,
                                                               np.float32)
  imp.weights["inception/logits/bias"] = b.astype(np.float32)
  return imp.weights


def load_weights(path):
  """The InceptionV3 weight dict of TF-GAN's frozen graph at `path` (the .pb, or the tarball as downloaded)."""
  return import_graph(parse_graph(read_graph_bytes(path)))


def main(argv=None):
  argv = sys.argv[1:] if argv is None else argv
  if len(argv) != 2:
    sys.stderr.write("usage: python -m compare_gan_b200.inception_graph SRC OUT.npz\n"
                     "  SRC: inceptionv1_for_inception_score.pb or frozen_inception_v1_2015_12_05.tar.gz\n")
    return 2
  weights = load_weights(argv[0])
  np.savez(argv[1], **weights)
  print("wrote %d arrays to %s; set CGAN_INCEPTION_NPZ to use them" % (len(weights), argv[1]))
  return 0


if __name__ == "__main__":
  sys.exit(main())
