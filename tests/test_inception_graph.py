"""Import of TF-GAN's frozen Inception GraphDef (`compare_gan_b200.inception_graph`).

The fixture is a GraphDef of the whole `inception.SPEC` topology in the 2015 graph's naming style (`conv`, `conv_1`,
`mixed/tower_1/conv_2`, `mixed/join`, `softmax/weights`), with random kernels and batch-norm constants.  It is written by
the minimal protobuf encoder below, independent of the module under test and of `tf_checkpoint`'s writer, and varies
what a real file may hold: both batch-norm ops, `scale_after_normalization` true and false, `Concat` and `ConcatV2`
(axis 3 and -1), Identity / CheckNumerics nodes with control inputs, `:0` input suffixes, weights behind `read`
Identities, off-path nodes the importer never interprets (a string constant, the pre-processing ops, Softmax), and
constants stored as `tensor_content`, packed / unpacked `float_val`, one- and two-value `float_val` fills and `int_val`.
A float64 numpy interpreter of the UNFOLDED fixture graph is the reference the imported (folded) weights are held to.
"""
import io
import os
import re
import struct
import subprocess
import sys
import tarfile

import numpy as np
import pytest
import torch

from compare_gan_b200 import inception, inception_graph
from oracle import inception as oinc
from tests.gpu_util import assert_close, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- minimal protobuf encoder ----------------------------------------------------------------------------------------

def _uv(v):
  v &= (1 << 64) - 1
  out = bytearray()
  while True:
    b, v = v & 0x7F, v >> 7
    out.append(b | (0x80 if v else 0))
    if not v:
      return bytes(out)


def _tag(field, wire):
  return _uv(field << 3 | wire)


def _ld(field, payload):
  return _tag(field, 2) + _uv(len(payload)) + payload


def _vf(field, v):
  return _tag(field, 0) + _uv(int(v))


def _ff(field, v):
  return _tag(field, 5) + struct.pack("<f", v)


def _tensor_proto(a, mode):
  """TensorProto of `a`; mode: content | packed | unpacked | fill (float_val holds a's first value, a is constant) |
  fill2 (float_val holds a's first two values, the rest equal the second) | int_packed | int_unpacked | string."""
  if mode == "string":
    return _vf(1, 7) + _ld(2, b"") + _ld(8, a)
  a = np.asarray(a)
  code = {np.dtype(np.float32): 1, np.dtype(np.int32): 3}[a.dtype]
  msg = _vf(1, code) + _ld(2, b"".join(_ld(2, _vf(1, d)) for d in a.shape))
  flat = a.ravel()
  if mode == "content":
    return msg + _ld(4, a.astype(a.dtype.newbyteorder("<")).tobytes())
  if mode == "packed":
    return msg + _ld(5, flat.astype("<f4").tobytes())
  if mode == "unpacked":
    return msg + b"".join(_ff(5, v) for v in flat)
  if mode in ("fill", "fill2"):
    head = flat[:1 if mode == "fill" else 2]
    assert (flat[len(head):] == head[-1]).all()
    return msg + _ld(5, head.astype("<f4").tobytes())
  if mode == "int_packed":
    return msg + _ld(7, b"".join(_uv(int(v)) for v in flat))
  assert mode == "int_unpacked"
  return msg + b"".join(_vf(7, v) for v in flat)


def _attr_value(kind, v, mode=None):
  if kind == "s":
    return _ld(2, v.encode())
  if kind == "i":
    return _vf(3, v)
  if kind == "f":
    return _ff(4, v)
  if kind == "b":
    return _vf(5, 1 if v else 0)
  if kind == "type":
    return _vf(6, v)
  if kind == "list_i":        # ListValue.i, packed or one entry per value
    body = _ld(3, b"".join(_uv(x) for x in v)) if mode == "packed" else b"".join(_vf(3, x) for x in v)
    return _ld(1, body)
  assert kind == "tensor"
  return _ld(8, _tensor_proto(v, mode))


def encode_graph(nodes):
  out = []
  for n in nodes:
    msg = _ld(1, n["name"].encode()) + _ld(2, n["op"].encode())
    msg += b"".join(_ld(3, s.encode()) for s in n["inputs"])
    for key, val in n["attr"].items():
      msg += _ld(5, _ld(1, key.encode()) + _ld(2, _attr_value(*val)))
    out.append(_ld(1, msg))
  return b"".join(out)


# ---- the fixture graph -----------------------------------------------------------------------------------------------

BN_KINDS = [("BatchNormWithGlobalNormalization", True), ("BatchNormWithGlobalNormalization", False),
            ("FusedBatchNorm", True), ("FusedBatchNormV2", True), ("FusedBatchNormV3", True)]


class GraphBuilder(object):

  def __init__(self, seed):
    self.rng = np.random.RandomState(seed)
    self.nodes, self.counts, self.nconv = [], {}, 0

  def add(self, name, op, inputs=(), **attr):
    self.nodes.append({"name": name, "op": op, "inputs": list(inputs), "attr": attr})
    return name

  def const(self, name, a, mode="content"):
    a = np.asarray(a)
    return self.add(name, "Const", value=("tensor", a, mode), dtype=("type", 1 if a.dtype == np.float32 else 3))

  def unique(self, scope, base):
    k = self.counts.get((scope, base), 0)
    self.counts[(scope, base)] = k + 1
    return (scope + "/" if scope else "") + (base if k == 0 else "%s_%d" % (base, k))

  def conv(self, scope, x, kh, kw, cin, cout, stride, padding):
    i, rng = self.nconv, self.rng
    self.nconv += 1
    name = self.unique(scope, "conv")
    w = (rng.standard_normal((kh, kw, cin, cout)) * np.sqrt(2.0 / (kh * kw * cin))).astype(np.float32)
    params = self.const(name + "/conv2d_params", w)
    if i % 7 == 3:
      params = self.add(name + "/conv2d_params/read", "Identity", [params])
    strides = ("list_i", [1, stride, stride, 1], "packed" if i % 2 else "unpacked")
    conv = self.add(name + "/Conv2D", "Conv2D", [x + (":0" if i % 9 == 4 else ""), params], T=("type", 1),
                    strides=strides, padding=("s", padding), data_format=("s", "NHWC"), use_cudnn_on_gpu=("b", True))
    # He-normal kernels keep E[x^2] through conv + ReLU; with E[gamma^2 / variance] ~ 1 the batch norms keep it too, so
    # activations stay O(1) through all 94 layers and the logits give a softmax that is not one-hot
    consts = {"mean": rng.standard_normal(cout) * 0.1, "variance": rng.uniform(0.8, 1.25, cout),
              "beta": rng.standard_normal(cout) * 0.1, "gamma": rng.uniform(0.8, 1.2, cout)}
    modes = dict.fromkeys(consts, "content")
    special = {0: ("mean", "packed"), 1: ("variance", "unpacked"), 2: ("beta", "fill"), 4: ("gamma", "fill2"),
               5: ("beta", "fill2"), 10: ("mean", "unpacked")}
    if i in special:
      key, mode = special[i]
      modes[key] = mode
      if mode == "fill":
        consts[key][:] = consts[key][0]
      elif mode == "fill2":
        consts[key][2:] = consts[key][1]
    c = {k: self.const(name + "/batchnorm/" + k, v.astype(np.float32), modes[k]) for k, v in consts.items()}
    op, scaled = BN_KINDS[i % len(BN_KINDS)]
    eps = [1e-3, 1e-5, 1e-4][i % 3]
    if op == "BatchNormWithGlobalNormalization":
      bn = self.add(name + "/batchnorm", op, [conv, c["mean"], c["variance"], c["beta"], c["gamma"]], T=("type", 1),
                    variance_epsilon=("f", eps), scale_after_normalization=("b", scaled))
    else:
      bn = self.add(name + "/batchnorm", op, [conv, c["gamma"], c["beta"], c["mean"], c["variance"]], T=("type", 1),
                    epsilon=("f", eps), is_training=("b", False), data_format=("s", "NHWC"))
    out = self.add(name, "Relu", [bn], T=("type", 1))
    if i % 11 == 5:
      out = self.add(name + "/check", "CheckNumerics", [out, "^" + c["beta"]], message=("s", "non-finite activation"))
    if i % 13 == 6:
      out = self.add(name + "/identity", "Identity", [out + ":0", "^" + conv])
    return out, cout

  def pool(self, scope, x, mode, k, s, padding, name=None):
    return self.add(name or self.unique(scope, "pool"), {"max": "MaxPool", "avg": "AvgPool"}[mode], [x], T=("type", 1),
                    ksize=("list_i", [1, k, k, 1], "unpacked"), strides=("list_i", [1, s, s, 1], "packed"),
                    padding=("s", padding), data_format=("s", "NHWC"))

  def concat(self, name, xs, op, axis):
    ax = self.const(name + "/concat_dim", np.array(axis, np.int32), "int_packed" if axis == 3 else "int_unpacked")
    inputs = [ax] + xs if op == "Concat" else xs + [ax]
    return self.add(name, op, inputs, N=("i", len(xs)), T=("type", 1))

  def seq(self, scope, items, x, c, concat_op):
    for it in items:
      if it[0] == "conv":
        _, _, cout, kh, kw, stride, padding = it
        x, c = self.conv(scope, x, kh, kw, c, cout, stride, padding)
      elif it[0] == "pool":
        x = self.pool(scope, x, *it[1:])
      elif it[0] == "split":
        sub = scope + "/mixed"
        outs = [self.seq(sub, br, x, c, concat_op) for br in it[1]]
        x = self.concat(sub, [o[0] for o in outs], concat_op, 3)
        c = sum(o[1] for o in outs)
      else:
        x, c = self.block(it[1], x, c, it[2])
    return x, c

  def block(self, name, x, c, branches):
    b = int(name.split("_")[1]) if "_" in name else 0
    op, inner = ("Concat", "ConcatV2") if b % 2 == 0 else ("ConcatV2", "Concat")
    outs, towers = [], 0
    for br in branches:
      if len(br) == 1 and br[0][0] != "split":
        scope = name
      else:
        scope = name + "/" + ("tower" if towers == 0 else "tower_%d" % towers)
        towers += 1
      outs.append(self.seq(scope, br, x, c, inner))
    axis = -1 if op == "ConcatV2" and b % 3 == 0 else 3
    return self.concat(name + "/join", [o[0] for o in outs], op, axis), sum(o[1] for o in outs)


def build_fixture(seed=0):
  """Node list of the fixture graph (see the module docstring)."""
  g = GraphBuilder(seed)
  g.add("DecodeJpeg/contents", "Const", value=("tensor", b"\xff\xd8 not decoded", "string"), dtype=("type", 7))
  g.add("ExpandDims", "Placeholder", dtype=("type", 1))
  g.add("Sub", "Sub", ["ExpandDims", g.const("Sub/y", np.float32(128.0))])
  g.add("Mul", "Mul", ["Sub", g.const("Mul/y", np.float32(1.0 / 128))])
  x, c = g.seq("", inception.SPEC, "Mul", 3, None)
  assert c == inception.POOL_DIM
  pool = g.pool("", x, "avg", inception_graph.FINAL_HW, 1, "VALID", name="pool_3")
  flat = g.add("pool_3/_reshape", "Reshape", [pool, g.const("pool_3/_reshape/shape", np.array([-1, 2048], np.int32))])
  w = (g.rng.standard_normal((inception.NUM_CLASSES, inception.POOL_DIM)) / np.sqrt(2048)).astype(np.float32)
  mm = g.add("softmax/logits/MatMul", "MatMul", [flat, g.const("softmax/weights", w)], transpose_a=("b", False),
             transpose_b=("b", True))
  bias = g.const("softmax/biases", (g.rng.standard_normal(inception.NUM_CLASSES) * 0.1).astype(np.float32), "packed")
  g.add("logits", "BiasAdd", [mm, bias], T=("type", 1), data_format=("s", "NHWC"))
  g.add("softmax", "Softmax", ["logits"])
  return g.nodes


# ---- float64 interpreter of the fixture graph ------------------------------------------------------------------------

def _same_pads(n, k, s):
  out = -(-n // s)
  total = max((out - 1) * s + k - n, 0)
  return total // 2, total - total // 2


def _windows(x, kh, kw, s, padding, fill):
  """[N, OH, OW, C, kh, kw] view of the TF padding of x (NHWC)."""
  if padding == "SAME":
    x = np.pad(x, ((0, 0), _same_pads(x.shape[1], kh, s), _same_pads(x.shape[2], kw, s), (0, 0)), constant_values=fill)
  return np.lib.stride_tricks.sliding_window_view(x, (kh, kw), axis=(1, 2))[:, ::s, ::s]


def _value(n):
  a = n["attr"]["value"][1]
  return a.astype(np.float64) if a.dtype == np.float32 else a


def interpret(nodes, images):
  """pool_3 [N, 2048] and logits [N, 1008] of the graph `nodes` fed `images` (float64 NHWC) as `Mul`."""
  vals = {"Mul": images}
  for n in nodes:
    op, at = n["op"], {k: v[1] for k, v in n["attr"].items()}
    if n["name"] == "Mul" or op in ("Placeholder", "Sub", "Softmax") or (op == "Const" and at["dtype"] == 7):
      continue
    if op == "Const":
      vals[n["name"]] = _value(n)
      continue
    xs = [vals[s.split(":")[0]] for s in n["inputs"] if not s.startswith("^")]
    if op == "Conv2D":
      w = xs[1]
      win = _windows(xs[0], w.shape[0], w.shape[1], at["strides"][1], at["padding"], 0.0)
      y = np.tensordot(win, w, axes=([3, 4, 5], [2, 0, 1]))
    elif op == "BatchNormWithGlobalNormalization":
      x, m, v, beta, gamma = xs
      y = (x - m) / np.sqrt(v + np.float64(np.float32(at["variance_epsilon"])))
      y = (y * gamma if at["scale_after_normalization"] else y) + beta
    elif op.startswith("FusedBatchNorm"):
      x, scale, offset, m, v = xs
      y = (x - m) / np.sqrt(v + np.float64(np.float32(at["epsilon"]))) * scale + offset
    elif op == "Relu":
      y = np.maximum(xs[0], 0.0)
    elif op in ("Identity", "CheckNumerics"):
      y = xs[0]
    elif op in ("MaxPool", "AvgPool"):
      k, s, pad = at["ksize"][1], at["strides"][1], at["padding"]
      if op == "MaxPool":
        y = _windows(xs[0], k, k, s, pad, -np.inf).max(axis=(4, 5))
      else:         # TF's SAME average divides by the number of cells inside the input
        y = _windows(xs[0], k, k, s, pad, 0.0).sum(axis=(4, 5)) / \
            _windows(np.ones_like(xs[0][..., :1]), k, k, s, pad, 0.0).sum(axis=(4, 5))
    elif op == "Concat":
      y = np.concatenate(xs[1:], axis=int(xs[0]))
    elif op == "ConcatV2":
      y = np.concatenate(xs[:-1], axis=int(xs[-1]))
    elif op == "Reshape":
      y = xs[0].reshape(xs[1])
    elif op == "MatMul":
      y = xs[0] @ (xs[1].T if at["transpose_b"] else xs[1])
    elif op == "BiasAdd":
      y = xs[0] + xs[1]
    else:
      raise AssertionError("the interpreter does not know op %s" % op)
    vals[n["name"]] = y
  return vals["pool_3"].reshape(-1, inception.POOL_DIM), vals["logits"]


# ---- fixtures --------------------------------------------------------------------------------------------------------

def _write(nodes, path):
  with open(path, "wb") as f:
    f.write(encode_graph(nodes))
  return path


@pytest.fixture(scope="module")
def fixture_graph(tmp_path_factory):
  """(nodes, .pb path, tarball path)."""
  d = tmp_path_factory.mktemp("inception_graph")
  nodes = build_fixture(0)
  pb = _write(nodes, str(d / inception_graph.GRAPH_MEMBER))
  tgz = str(d / "frozen_inception_v1_2015_12_05.tar.gz")
  with tarfile.open(tgz, "w:gz", compresslevel=1) as tar:
    tar.add(pb, arcname=inception_graph.GRAPH_MEMBER)
    info = tarfile.TarInfo("imagenet_comp_graph_label_strings.txt")
    labels = b"dummy\n" * 1008
    info.size = len(labels)
    tar.addfile(info, io.BytesIO(labels))
  return nodes, pb, tgz


@pytest.fixture(scope="module")
def imported(fixture_graph):
  return inception_graph.load_weights(fixture_graph[1])


def _images(n=2, seed=2):
  return np.random.RandomState(seed).rand(n, 299, 299, 3).astype(np.float32) * 2 - 1


# ---- CPU -------------------------------------------------------------------------------------------------------------

def test_fixture_exercises_every_encoding(fixture_graph):
  nodes = fixture_graph[0]
  ops = {n["op"] for n in nodes}
  assert set(op for op, _ in BN_KINDS) <= ops and {"Concat", "ConcatV2", "CheckNumerics", "Identity"} <= ops
  bnwgn = [n["attr"]["scale_after_normalization"][1] for n in nodes if n["op"] == "BatchNormWithGlobalNormalization"]
  assert True in bnwgn and False in bnwgn
  modes = [n["attr"]["value"][2] for n in nodes if n["op"] == "Const"]
  assert modes.count("content") > 300
  for m in ("packed", "unpacked", "fill", "fill2", "int_packed", "int_unpacked", "string"):
    assert m in modes, m
  assert any(s.startswith("^") for n in nodes for s in n["inputs"])
  assert any(s.endswith(":0") for n in nodes for s in n["inputs"])


def test_imported_weights_match_the_unfolded_graph_in_float64(fixture_graph, imported):
  """The oracle network on the imported (BN-folded, fp32-rounded) weights against the float64 interpretation of the
  graph itself: the fp32 rounding of the folded weights is the only difference."""
  x = _images().astype(np.float64)
  ref_pool, ref_logits = interpret(fixture_graph[0], x)
  w64 = {k: torch.from_numpy(v.astype(np.float64)) for k, v in imported.items()}
  pool, logits = oinc.inception_v3(torch.from_numpy(x), w64)
  e_pool, e_logits = rel_err(pool.numpy(), ref_pool), rel_err(logits.numpy(), ref_logits)
  print("imported vs unfolded graph, float64: pool_3 rel-L2 %.2e, logits rel-L2 %.2e (pool_3 rms %.3f, logits std %.3f)"
        % (e_pool, e_logits, np.sqrt(np.mean(ref_pool ** 2)), np.std(ref_logits)))
  for a in (ref_pool, ref_logits):                # the random network neither collapsed nor blew up
    assert 0.05 < np.sqrt(np.mean(a ** 2)) < 20
  assert e_pool <= 1e-5 and e_logits <= 1e-5


def test_pb_and_tarball_import_alike_with_the_synthetic_key_space(fixture_graph, imported):
  from_tar = inception_graph.load_weights(fixture_graph[2])
  synth = inception.synthetic_weights(0)
  assert sorted(imported) == sorted(synth) == sorted(from_tar)
  for k, v in synth.items():
    assert imported[k].shape == v.shape and imported[k].dtype == np.float32, k
    np.testing.assert_array_equal(imported[k], from_tar[k], err_msg=k)


def test_converter_cli_writes_the_npz_the_extractor_reads(fixture_graph, imported, tmp_path):
  out = str(tmp_path / "inception.npz")
  env = dict(os.environ, PYTHONPATH=ROOT)
  subprocess.run([sys.executable, "-m", "compare_gan_b200.inception_graph", fixture_graph[2], out], cwd=ROOT, env=env,
                 check=True, capture_output=True)
  data = np.load(out)
  assert sorted(data.files) == sorted(imported)
  for k in data.files:
    np.testing.assert_array_equal(data[k], imported[k], err_msg=k)
  bad = subprocess.run([sys.executable, "-m", "compare_gan_b200.inception_graph", fixture_graph[2]], cwd=ROOT, env=env,
                       capture_output=True)
  assert bad.returncode == 2 and b"usage" in bad.stderr


def _node(nodes, name):
  return next(n for n in nodes if n["name"] == name)


def _with(nodes, name, op=None, inputs=None, **attr):
  """A copy of `nodes` with node `name` changed."""
  nodes = list(nodes)
  i = nodes.index(_node(nodes, name))
  n = dict(nodes[i], attr=dict(nodes[i]["attr"], **attr))
  if op is not None:
    n["op"] = op
  if inputs is not None:
    n["inputs"] = inputs
  nodes[i] = n
  return nodes


def _swap_branches(nodes):
  ins = list(_node(nodes, "mixed_1/join")["inputs"])
  k = 0 if _node(nodes, "mixed_1/join")["op"] == "ConcatV2" else 1
  ins[k], ins[k + 1] = ins[k + 1], ins[k]
  return _with(nodes, "mixed_1/join", inputs=ins)


def _drop_branch(nodes):
  n = _node(nodes, "mixed_4/join")
  ins = [s for s in n["inputs"] if "tower_1" not in s]
  return _with(nodes, "mixed_4/join", inputs=ins, N=("i", n["attr"]["N"][1] - 1))


def _thousand_classes(nodes):
  rng = np.random.RandomState(5)
  nodes = _with(nodes, "softmax/weights", value=("tensor", rng.standard_normal((1000, 2048)).astype(np.float32), "content"))
  return _with(nodes, "softmax/biases", value=("tensor", np.zeros(1000, np.float32), "content"))


MUTATIONS = {
    "stride": (lambda g: _with(g, "mixed_3/conv/Conv2D", strides=("list_i", [1, 1, 1, 1], "packed")),
               "mixed_3/conv/Conv2D"),
    "padding": (lambda g: _with(g, "conv_1/Conv2D", padding=("s", "SAME")), "conv_1/Conv2D"),
    "swapped_branches": (_swap_branches, "mixed_1/join"),
    "removed_branch": (_drop_branch, "mixed_4/join"),
    "unknown_op": (lambda g: _with(g, "mixed_5/tower_1/conv_2", op="Relu6"), "mixed_5/tower_1/conv_2"),
    "nchw": (lambda g: _with(g, "mixed_7/conv/Conv2D", data_format=("s", "NCHW")), "mixed_7/conv/Conv2D"),
    "1000_classes": (_thousand_classes, "softmax/logits/MatMul"),
}


@pytest.mark.parametrize("case", sorted(MUTATIONS))
def test_a_graph_that_is_not_spec_raises_naming_the_node(fixture_graph, case):
  mutate, name = MUTATIONS[case]
  nodes = inception_graph.parse_graph(encode_graph(mutate(fixture_graph[0])))
  with pytest.raises(ValueError, match=re.escape(repr(name))) as e:
    inception_graph.import_graph(nodes)
  print(case, "->", e.value)
  assert "SPEC" in str(e.value)


def test_tensor_decoding_edge_cases():
  """float_val fills (one value, two values, none = zeros), int_val signs, and a too-long float_val."""
  dec = inception_graph._tensor
  proto = lambda a, mode: _tensor_proto(np.asarray(a), mode)
  np.testing.assert_array_equal(dec(proto(np.full((2, 3), 0.5, np.float32), "fill"), "t"), np.full((2, 3), 0.5))
  np.testing.assert_array_equal(dec(proto(np.float32([1, 2, 2, 2]), "fill2"), "t"), [1, 2, 2, 2])
  np.testing.assert_array_equal(dec(proto(np.float32([1, -2.5]), "unpacked"), "t"), [1, -2.5])
  assert dec(_vf(1, 1) + _ld(2, _ld(2, _vf(1, 4))), "t").tolist() == [0, 0, 0, 0]
  np.testing.assert_array_equal(dec(proto(np.int32([-1, 2048]), "int_unpacked"), "t"), [-1, 2048])
  np.testing.assert_array_equal(dec(proto(np.int32([-7, 3]), "int_packed"), "t"), [-7, 3])
  too_long = _vf(1, 1) + _ld(2, _ld(2, _vf(1, 1))) + _ld(5, np.float32([1, 2]).tobytes())
  with pytest.raises(ValueError, match="2 values for tensor shape"):
    dec(too_long, "t")


def test_tarball_without_the_graph_member_raises(tmp_path):
  path = str(tmp_path / "other.tar")
  with tarfile.open(path, "w") as tar:
    info = tarfile.TarInfo("README")
    tar.addfile(info)
  with pytest.raises(ValueError, match=inception_graph.GRAPH_MEMBER):
    inception_graph.load_weights(path)


# ---- GPU -------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_inception_v3_on_imported_weights(imported):
  """The engine's InceptionV3 on the imported weights against the oracle, within test_inception_v3_features'
  (fp32, 2e-4) and test_inception_v3_features_tf32's (math_mode 1: 2e-3 / 3e-3) bounds."""
  from compare_gan_b200 import kernels as K
  K.init(0)
  x = _images()
  rp, rl = oinc.inception_v3(x, imported)
  pool, logits = inception.InceptionV3(imported)(K.from_numpy(x))
  print("fp32: pool_3 %.2e logits %.2e" % (rel_err(pool.cpu(), rp.numpy()), rel_err(logits.cpu(), rl.numpy())))
  assert_close(pool.cpu(), rp.numpy(), 2e-4, "pool_3")
  assert_close(logits.cpu(), rl.numpy(), 2e-4, "logits")
  K.set_math_mode(1)
  try:
    pool, logits = inception.InceptionV3(imported)(K.from_numpy(x))
  finally:
    K.set_math_mode(0)
  print("tf32: pool_3 %.2e logits %.2e" % (rel_err(pool.cpu(), rp.numpy()), rel_err(logits.cpu(), rl.numpy())))
  assert_close(pool.cpu(), rp.numpy(), 2e-3, "pool_3 (tf32)")
  assert_close(logits.cpu(), rl.numpy(), 3e-3, "logits (tf32)")


@pytest.mark.gpu
def test_evaluate_on_the_converted_npz(fixture_graph, tmp_path, monkeypatch):
  """`evaluate` with $CGAN_INCEPTION_NPZ set to the converter's output: FID / IS / KID equal to the oracle's with the
  same weights (as test_eval_fid_is_kid_against_oracle checks), and no `inception_weights_synthetic` stamp."""
  from compare_gan_b200 import eval_gan_lib, eval_utils
  from compare_gan_b200 import kernels as K
  from compare_gan_b200.metrics import fid_score, inception_score, kid_score
  from oracle import metrics as ometrics
  from tests.gpu_util import make_pair
  K.init(0)
  out = str(tmp_path / "inception.npz")
  assert inception_graph.main([fixture_graph[2], out]) == 0
  monkeypatch.setenv("CGAN_INCEPTION_NPZ", out)
  saved = dict(eval_utils._INCEPTION)
  eval_utils._INCEPTION.clear()
  try:
    net = eval_utils.get_inception()
    assert not net.synthetic
    w = net.host_weights
    data = np.load(out)
    for k in data.files:
      np.testing.assert_array_equal(w[k], data[k], err_msg=k)
    eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True)
    tasks = [fid_score.FIDScoreTask(), inception_score.InceptionScoreTask(), kid_score.KIDScoreTask()]
    n = 96
    real = np.random.RandomState(3).rand(n, 32, 32, 3).astype(np.float32)
    res = eval_gan_lib.evaluate(eng, tasks, num_averaging_runs=1, num_samples=n, batch_size=32, seed=42,
                                real_images=real)
    assert "inception_weights_synthetic" not in res
    rs = np.random.RandomState(42)
    fake_acts, fake_logits = [], []
    for _ in range(n // 32):
      imgs = eval_gan_lib.generate_batch(eng, 32, rs).cpu()
      p, l = oinc.inception_v3(oinc.preprocess(imgs), w)
      fake_acts.append(p.numpy())
      fake_logits.append(l.numpy())
    ra = oinc.inception_v3(oinc.preprocess(real), w)[0].numpy()
    fa, fl = np.concatenate(fake_acts), np.concatenate(fake_logits)
    p = np.exp(fl - fl.max(1, keepdims=True))
    assert (p.max(1) / p.sum(1)).mean() < 0.5          # class posteriors that are not one-hot
    fid_ref = ometrics.compute_fid_from_activations(ra, fa)
    is_ref = ometrics.inception_score_from_logits(fl)
    kid_ref = ometrics.kid(fa, ra)
    print("FID %.6f (oracle %.6f), IS %.6f (oracle %.6f), KID %.3e (oracle %.3e)"
          % (res["fid_score_mean"], fid_ref, res["inception_score_mean"], is_ref, res["kid_score_mean"], kid_ref))
    assert abs(res["fid_score_mean"] - fid_ref) <= 5e-3 * abs(fid_ref), (res["fid_score_mean"], fid_ref)
    assert abs(res["inception_score_mean"] - is_ref) <= 5e-3 * abs(is_ref), (res["inception_score_mean"], is_ref)
    assert abs(res["kid_score_mean"] - kid_ref) <= 5e-3 * abs(kid_ref) + 1e-6, (res["kid_score_mean"], kid_ref)
  finally:
    eval_utils._INCEPTION.clear()
    eval_utils._INCEPTION.update(saved)
