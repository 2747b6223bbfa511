"""Inception-v3 (2015 classify_image graph) feature extractor built from the engine's own conv / pooling kernels.

The reference obtains `pool_3:0` (2048-d) and `logits:0` (1008-d) from TF-GAN's frozen graph
(`eval_utils.py:41-49, 165-175`; tfgan.eval.run_inception).  That graph is downloaded at run time and is not
available offline, so the WEIGHTS here are deterministic synthetic values (He-normal, BN folded into a per-channel
bias) of the exact topology — throughput and the FID/IS arithmetic are exercised faithfully, absolute scores versus the
real Inception are "parity unpinned" (SURVEY.md §7 item 7).  `load_weights` accepts a real weight dict
(`inception/<layer>/kernel|bias`, HWIO) when one is available; `inception_graph.py` makes one from TF-GAN's frozen graph.
"""
import numpy as np

from . import kernels as K
from . import tape

# (name, cout, kh, kw, stride, padding) helpers ------------------------------------------------------------------


def _conv(name, cout, kh, kw=None, stride=1, padding="SAME"):
  return ("conv", name, cout, kh, kh if kw is None else kw, stride, padding)


def inception_a(prefix, pool_features):
  return ("block", prefix, [
      [_conv("b1x1", 64, 1)],
      [_conv("b5x5_1", 48, 1), _conv("b5x5_2", 64, 5)],
      [_conv("b3x3dbl_1", 64, 1), _conv("b3x3dbl_2", 96, 3), _conv("b3x3dbl_3", 96, 3)],
      [("pool", "avg", 3, 1, "SAME"), _conv("bpool", pool_features, 1)],
  ])


def inception_b(prefix):
  return ("block", prefix, [
      [_conv("b3x3", 384, 3, stride=2, padding="VALID")],
      [_conv("b3x3dbl_1", 64, 1), _conv("b3x3dbl_2", 96, 3), _conv("b3x3dbl_3", 96, 3, stride=2, padding="VALID")],
      [("pool", "max", 3, 2, "VALID")],
  ])


def inception_c(prefix, c7):
  return ("block", prefix, [
      [_conv("b1x1", 192, 1)],
      [_conv("b7x7_1", c7, 1), _conv("b7x7_2", c7, 1, 7), _conv("b7x7_3", 192, 7, 1)],
      [_conv("b7x7dbl_1", c7, 1), _conv("b7x7dbl_2", c7, 7, 1), _conv("b7x7dbl_3", c7, 1, 7),
       _conv("b7x7dbl_4", c7, 7, 1), _conv("b7x7dbl_5", 192, 1, 7)],
      [("pool", "avg", 3, 1, "SAME"), _conv("bpool", 192, 1)],
  ])


def inception_d(prefix):
  return ("block", prefix, [
      [_conv("b3x3_1", 192, 1), _conv("b3x3_2", 320, 3, stride=2, padding="VALID")],
      [_conv("b7x7x3_1", 192, 1), _conv("b7x7x3_2", 192, 1, 7), _conv("b7x7x3_3", 192, 7, 1),
       _conv("b7x7x3_4", 192, 3, stride=2, padding="VALID")],
      [("pool", "max", 3, 2, "VALID")],
  ])


def inception_e(prefix, pool_mode):
  return ("block", prefix, [
      [_conv("b1x1", 320, 1)],
      [_conv("b3x3_1", 384, 1), ("split", [[_conv("b3x3_2a", 384, 1, 3)], [_conv("b3x3_2b", 384, 3, 1)]])],
      [_conv("b3x3dbl_1", 448, 1), _conv("b3x3dbl_2", 384, 3),
       ("split", [[_conv("b3x3dbl_3a", 384, 1, 3)], [_conv("b3x3dbl_3b", 384, 3, 1)]])],
      [("pool", pool_mode, 3, 1, "SAME"), _conv("bpool", 192, 1)],
  ])


SPEC = [
    _conv("conv_1a", 32, 3, stride=2, padding="VALID"),
    _conv("conv_2a", 32, 3, padding="VALID"),
    _conv("conv_2b", 64, 3),
    ("pool", "max", 3, 2, "VALID"),
    _conv("conv_3b", 80, 1),
    _conv("conv_4a", 192, 3, padding="VALID"),
    ("pool", "max", 3, 2, "VALID"),
    inception_a("mixed", 32), inception_a("mixed_1", 64), inception_a("mixed_2", 64),
    inception_b("mixed_3"),
    inception_c("mixed_4", 128), inception_c("mixed_5", 160), inception_c("mixed_6", 160), inception_c("mixed_7", 192),
    inception_d("mixed_8"),
    inception_e("mixed_9", "avg"),
    inception_e("mixed_10", "max"),     # the 2015 graph max-pools in its last block
]
NUM_CLASSES = 1008
POOL_DIM = 2048


def walk_convs(spec=SPEC, cin=3, prefix=""):
  """Yields (full_name, kh, kw, cin, cout) in definition order and returns nothing; used to create weights."""
  out = []

  def seq(items, c, pre):
    for it in items:
      if it[0] == "conv":
        _, name, cout, kh, kw, _, _ = it
        out.append((pre + name, kh, kw, c, cout))
        c = cout
      elif it[0] == "split":
        c = sum(seq(br, c, pre) for br in it[1])
      elif it[0] == "block":
        c = sum(seq(br, c, pre + it[1] + "/") for br in it[2])
    return c
  seq(spec, cin, prefix)
  return out


def _channels(items, c):
  """Output channels of a branch given its input channels."""
  for it in items:
    if it[0] == "conv":
      c = it[2]
    elif it[0] == "split":
      c = sum(_channels(br, c) for br in it[1])
    elif it[0] == "block":
      c = sum(_channels(br, c) for br in it[2])
  return c


def synthetic_weights(seed=0):
  """Deterministic He-normal weights (BN folded into a small bias) for the exact topology."""
  rng = np.random.RandomState(seed)
  w = {}
  for name, kh, kw, cin, cout in walk_convs():
    std = np.sqrt(2.0 / (kh * kw * cin))
    w["inception/%s/kernel" % name] = (rng.standard_normal((kh, kw, cin, cout)) * std).astype(np.float32)
    w["inception/%s/bias" % name] = (rng.standard_normal(cout) * 0.05).astype(np.float32)
  w["inception/logits/kernel"] = (rng.standard_normal((POOL_DIM, NUM_CLASSES)) / np.sqrt(POOL_DIM)).astype(np.float32)
  w["inception/logits/bias"] = np.zeros(NUM_CLASSES, np.float32)
  return w


def flops_per_image(size=299):
  """2*MAC of all convolutions + the logits layer for one `size` x `size` image."""
  total = [0]

  def seq(items, c, hw):
    for it in items:
      if it[0] == "conv":
        _, _, cout, kh, kw, s, pad = it
        hw = -(-hw // s) if pad == "SAME" else (hw - kh) // s + 1     # kh==kw whenever stride>1 / VALID here
        total[0] += 2 * hw * hw * kh * kw * c * cout
        c = cout
      elif it[0] == "pool":
        _, _, k, s, pad = it
        hw = -(-hw // s) if pad == "SAME" else (hw - k) // s + 1
      elif it[0] == "split":
        c = sum(seq(br, c, hw)[0] for br in it[1])
      elif it[0] == "block":
        res = [seq(br, c, hw) for br in it[2]]
        c, hw = sum(r[0] for r in res), res[0][1]
    return c, hw
  seq(SPEC, 3, size)
  return total[0] + 2 * POOL_DIM * NUM_CLASSES


class InceptionV3(object):

  def __init__(self, weights=None, seed=0):
    self.load_weights(weights if weights is not None else synthetic_weights(seed))

  def load_weights(self, weights):
    self.host_weights = weights
    self.w = {k: K.from_numpy(v) for k, v in weights.items()}

  def _seq(self, items, x, pre, sink=None, off=0):
    """Runs `items` on x.  With `sink` the LAST item stores into channels [off, ...) of the sink (the enclosing concat):
    convolutions write their slice directly (strided epilogue), pooling branches are copied in."""
    for i, it in enumerate(items):
      last = sink is not None and i == len(items) - 1
      if it[0] == "conv":
        _, name, _, _, _, stride, padding = it
        x = K.conv2d_relu(x, self.w["inception/%s%s/kernel" % (pre, name)], self.w["inception/%s%s/bias" % (pre, name)],
                          stride=stride, padding=padding, sink=sink if last else None, sink_off=off)
      elif it[0] == "pool":
        _, mode, k, s, pad = it
        x = K.pool2d(x, k, s, pad, mode)
        if last:
          sink.put(x, off)
          x = None
      elif it[0] in ("split", "block"):
        branches, bpre = (it[1], pre) if it[0] == "split" else (it[2], pre + it[1] + "/")
        cin = x.shape[3]
        widths = [_channels(br, cin) for br in branches]
        tgt, base = (sink, off) if last else (K.ChannelSink(sum(widths)), 0)
        for br, wd in zip(branches, widths):
          self._seq(br, x, bpre, tgt, base)
          base += wd
        x = None if last else tgt.buf
    return x

  def __call__(self, images):
    """images: [N,299,299,3] already scaled to [-1,1].  Returns (pool_3 [N,2048], logits [N,1008])."""
    with tape.no_record():
      x = self._seq(SPEC, images, "")
      pool = K.globalpool(x, mean=True)
      logits = K.bias_add(K.matmul(pool, self.w["inception/logits/kernel"]), self.w["inception/logits/bias"])
    return pool, logits
