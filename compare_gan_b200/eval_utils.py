"""Evaluation helpers (reference eval_utils.py:56-206): Inception features of image batches, on the GPU."""
import numpy as np
import torch

from . import inception
from . import kernels as K
from .tape import DT

NAN_DETECTED = 31337.0     # reference eval_gan_lib.py:40


class NanFoundError(Exception):
  """reference eval_utils.py:52-53."""


class EvalDataSample(object):
  """Container for a (fake or real) evaluation set (reference eval_utils.py:56-84), extended with the streaming
  FID moments accumulated on the device.  For a generated set `images` holds the first N samples (N = the largest
  images_needed of the evaluation's tasks, in [0, 255], on the device), not the whole set; None when no task needs them."""

  def __init__(self, images=None):
    self._images = images
    self.activations = None
    self.logits = None
    self.moments = None          # (mu, sigma) float64 from the device accumulator
    self._num_examples = None

  @property
  def images(self):
    return self._images

  def set_inception_features(self, activations, logits):
    self.activations, self.logits = activations, logits

  def set_num_examples(self, n):
    self._num_examples = n
    if self.activations is not None:
      self.activations = self.activations[:n]
    if self.logits is not None:
      self.logits = self.logits[:n]

  def discard_images(self):
    self._images = None


_INCEPTION = {}


def get_inception():
  """The Inception-v3 feature extractor of the metrics.  Real weights (the frozen TF-GAN graph's tensors in this package's
  key space, `inception/<layer>/kernel|bias`) are read from the .npz named by $CGAN_INCEPTION_NPZ; without it the
  extractor runs on deterministic SYNTHETIC weights of the exact topology (the graph cannot be downloaded here,
  reference eval_utils.py:41-49) — throughput is then real, the FID / IS values are not comparable with published ones."""
  import os
  dev = K._RT["device"]
  if dev not in _INCEPTION:
    path = os.environ.get("CGAN_INCEPTION_NPZ")
    weights = None
    if path:
      data = np.load(path)
      weights = {k: np.asarray(data[k], np.float32) for k in data.files}
    net = inception.InceptionV3(weights)
    net.synthetic = weights is None
    _INCEPTION[dev] = net
  return _INCEPTION[dev]


class FeatureAccumulator(object):
  """Streaming float64 (n, sum x, sum x x^T) on the device (cgan_cov_accumulate) + host copies of pool_3 / logits."""

  def __init__(self, dim=inception.POOL_DIM, keep_features=True):
    dev = K._RT["device"]
    self.dim, self.n, self.keep = dim, 0, keep_features
    self.s = torch.zeros(dim, dtype=torch.float64, device=dev)
    self.sxx = torch.zeros(dim, dim, dtype=torch.float64, device=dev)
    self.acts, self.logits = [], []

  def add(self, pool, logits, valid):
    """pool: [B,2048] DT, logits: [B,1008] DT; only the first `valid` rows count (last partial batch)."""
    K._call("cov_accumulate", pool.ptr, int(valid), self.dim, self.s.data_ptr(), self.sxx.data_ptr())
    self.n += int(valid)
    if self.keep:
      self.acts.append(pool.t[:valid].clone())
      self.logits.append(logits.t[:valid].clone())

  def finish(self, sample):
    from .metrics import fid_score
    from .tpu import tpu_ops
    if tpu_ops.num_replicas() > 1:          # sharded eval: final all-reduce of the statistics (SURVEY §8e)
      import torch.distributed as dist
      cnt = torch.tensor([float(self.n)], dtype=torch.float64, device=self.s.device)
      for t in (self.s, self.sxx, cnt):
        dist.all_reduce(t)
      self.n = int(cnt.item())
    sample.moments = fid_score.moments_from_sums(self.s.cpu().numpy(), self.sxx.cpu().numpy(), self.n)
    if self.keep:
      acts, logits = torch.cat(self.acts), torch.cat(self.logits)
      if tpu_ops.num_replicas() > 1:        # IS / KID need every sample's features: gather the shards (padded to equal length)
        acts, logits = _gather_rows(acts), _gather_rows(logits)
      sample.set_inception_features(acts.cpu().numpy(), logits.cpu().numpy())
    return sample


def _gather_rows(t):
  """all_gather of a [n_local, d] tensor whose n_local may differ by rank; rows come back in rank order."""
  import torch.distributed as dist
  world = dist.get_world_size()
  n = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
  counts = [torch.zeros_like(n) for _ in range(world)]
  dist.all_gather(counts, n)
  counts = [int(c.item()) for c in counts]
  pad = torch.zeros(max(counts), t.shape[1], dtype=t.dtype, device=t.device)
  pad[:t.shape[0]] = t
  parts = [torch.zeros_like(pad) for _ in range(world)]
  dist.all_gather(parts, pad)
  return torch.cat([p[:c] for p, c in zip(parts, counts)])


def inception_transform(images01):
  """images01: [B,h,w,c] DT in [0,1] (c = 1 is tiled to 3).  Returns (pool_3, logits) DTs
  (reference inception_transform, eval_utils.py:165-175: x*255, bilinear 299x299, (x-128)/128, Inception)."""
  if images01.shape[3] == 1:
    images01 = K.concat_channels([images01, images01, images01])
  x = K.resize_bilinear(images01, 299, 299, inception_scale=True)
  return get_inception()(x)


def inception_transform_np(images255, batch_size, keep_features=True):
  """reference eval_utils.py:178-206 (images in [0,255], numpy) -> EvalDataSample-ready accumulator."""
  acc = FeatureAccumulator(keep_features=keep_features)
  n = images255.shape[0]
  for i in range(0, n, batch_size):
    chunk = images255[i:i + batch_size].astype(np.float32) / 255.0
    valid = chunk.shape[0]
    if valid < batch_size:
      chunk = np.concatenate([chunk, np.zeros((batch_size - valid,) + chunk.shape[1:], np.float32)])
    pool, logits = inception_transform(K.from_numpy(chunk))
    acc.add(pool, logits, valid)
  return acc
