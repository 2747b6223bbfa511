"""Evaluation of a trained GAN (reference eval_gan_lib.py:65-212): sample the generator in inference mode in batches
of 64, run Inception on the samples, compute FID / IS / KID (and MS-SSIM on the first generated samples when a task asks
for images).  Everything up to the [N,2048] statistics stays on the GPU; sample generation can be sharded across ranks
with a final all-reduce of the statistics."""
import time

import numpy as np
import torch

from . import eval_utils
from . import kernels as K
from . import tape
from . import variables as V
from .runner_lib import eval_z_generator
from .tpu import tpu_ops

NAN_DETECTED = eval_utils.NAN_DETECTED


def _update_bn_accumulators(gan, batch_size, num_accu_examples=204800, rng=None):
  """reference eval_gan_lib.py:65-92: fill accu_mean/accu_variance by running G with update_accus=1 for
  num_accu_examples // batch_size batches.  The reference loads a fresh module per evaluation, i.e. its accumulators
  start at (0, 0, 1e-12): they are reset here so that repeated evaluations of one object do not average in the
  statistics of older weights."""
  accus = [v for k, v in gan.store.vars.items() if k.endswith("accu/update_accus")]
  if not accus:
    return False
  rng = rng or np.random
  for k, v in gan.store.vars.items():
    if k.endswith("accu/accu_mean") or k.endswith("accu/accu_variance"):
      K.fill_(v, 0.0)
    elif k.endswith("accu/accu_counter"):
      K.fill_(v, 1e-12)
  for v in accus:
    K.fill_(v, 1.0)
  for _ in range(num_accu_examples // batch_size):
    generate_batch(gan, batch_size, rng)
  for v in accus:
    K.fill_(v, 0.0)
  return True


def generate_batch(gan, batch_size, rng):
  """One inference-mode G call (z from gin `eval_z`, labels ~ U{0..C-1}, reference :127-146)."""
  z = K.from_numpy(eval_z_generator((batch_size, gan._z_dim), rng=rng))
  y = None
  if gan.conditional:
    labels = rng.randint(0, gan._dataset.num_classes, batch_size).astype(np.int32)
    y = K.one_hot(tape.DT(torch.from_numpy(labels).to(z.t.device)), gan._dataset.num_classes)
  with V.use(gan.store), tape.no_record():
    return gan.generator(z, y=y, is_training=False)


class use_ema_weights(object):
  """Evaluate G with its EMA shadow (reference modular_gan.py:266-285 exports the hub module with the EMA getter)."""

  def __init__(self, gan):
    self.gan = gan

  def __enter__(self):
    g = self.gan
    if g.ema is not None:
      self.saved = g.flat_g["param"].t.clone()
      K.copy_(g.flat_g["param"], g.ema)
    return self

  def __exit__(self, *a):
    g = self.gan
    if g.ema is not None:
      g.flat_g["param"].t.copy_(self.saved)


class _EvalBatchGraph(object):
  """`fuse` evaluation batches — inference-mode G, bilinear resize, Inception, float64 statistics update — captured into
  ONE CUDA graph (~330 kernel launches per batch would otherwise be paid in Python on every batch).  The reference
  evaluates in batches of 64 (eval_gan_lib.py:113); in inference mode every sample is independent of its batch mates
  (moving averages / accumulators, no batch statistics), so running `fuse` consecutive batches as one device batch gives
  bit-identical features while the 17x17 and 8x8 Inception stages get `fuse` times as many pixel tiles per launch (at 64
  images they expose 145 / 32 tiles to 132 SMs).  The z / label stream is still drawn batch by batch in the same order."""

  def __init__(self, gan, batch_size, acc, fuse=1, keep_images=False):
    dev = K._RT["device"]
    self.ref_b, self.fuse = batch_size, fuse
    self.keep_images, self.images = keep_images, None
    batch_size = batch_size * fuse
    self.gan, self.b, self.acc = gan, batch_size, acc
    self.z = tape.DT(torch.zeros(batch_size, gan._z_dim, device=dev))
    self.labels = tape.DT(torch.zeros(batch_size, dtype=torch.int32, device=dev)) if gan.conditional else None
    self.pool = tape.DT(torch.zeros(batch_size, eval_utils.inception.POOL_DIM, device=dev))
    self.logits = tape.DT(torch.zeros(batch_size, eval_utils.inception.NUM_CLASSES, device=dev))
    snap_s, snap_sxx = acc.s.clone(), acc.sxx.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      K.sync_stream()
      for _ in range(2):
        self._body()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    self.graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(self.graph):
      K.sync_stream()
      self._body()
    K.sync_stream()
    torch.cuda.synchronize()
    acc.s.copy_(snap_s)
    acc.sxx.copy_(snap_sxx)

  def _body(self):
    g = self.gan
    y = K.one_hot(self.labels, g._dataset.num_classes) if g.conditional else None
    with V.use(g.store), tape.no_record():
      imgs = g.generator(self.z, y=y, is_training=False)
    if self.keep_images:      # G's output in a persistent buffer (allocated by the warm-up, before capture)
      if self.images is None:
        self.images = K.empty(*imgs.shape)
      K.copy_(self.images, imgs)
    pool, logits = eval_utils.inception_transform(imgs)
    K._call("cov_accumulate", pool.ptr, self.b, self.acc.dim, self.acc.s.data_ptr(), self.acc.sxx.data_ptr())
    K.copy_(self.pool, pool)
    K.copy_(self.logits, logits)

  def run_batches(self, rng, num_batches, keeper):
    """Draws the latents of all batches first (same RNG order as the eager path: z then labels, batch by batch), ships
    them to the device in one copy, then replays the graph back to back with no host synchronisation in between."""
    g = self.gan
    zs, ls = [], []
    for _ in range(num_batches):
      zpart, lpart = [], []
      for _ in range(self.fuse):        # reference order: z of a batch of `ref_b`, then its labels
        zpart.append(eval_z_generator((self.ref_b, g._z_dim), rng=rng))
        if g.conditional:
          lpart.append(rng.randint(0, g._dataset.num_classes, self.ref_b).astype(np.int32))
      zs.append(np.concatenate(zpart))
      if g.conditional:
        ls.append(np.concatenate(lpart))
    dev = self.z.t.device
    z_all = torch.from_numpy(np.stack(zs)).pin_memory().to(dev, non_blocking=True)
    l_all = torch.from_numpy(np.stack(ls)).pin_memory().to(dev, non_blocking=True) if g.conditional else None
    for i in range(num_batches):
      self.z.t.copy_(z_all[i], non_blocking=True)
      if g.conditional:
        self.labels.t.copy_(l_all[i], non_blocking=True)
      self.graph.replay()
      self.acc.n += self.b
      if self.images is not None:
        keeper.add(self.images)
      if self.acc.keep:     # device-side copies; one device->host transfer at finish()
        self.acc.acts.append(self.pool.t.clone())
        self.acc.logits.append(self.logits.t.clone())


class _ImageKeeper(object):
  """The first `n` generated images of one averaging run, kept on the device for the tasks that read images (MS-SSIM)."""

  def __init__(self, n):
    self.n, self.parts, self.have = n, [], 0

  def add(self, imgs, valid=None):
    take = min(self.n - self.have, imgs.shape[0] if valid is None else valid)
    if take > 0:
      self.parts.append(imgs.t[:take].clone())
      self.have += take

  def images255(self):
    if not self.parts:
      return None
    with tape.no_record():
      return K.affine(tape.DT(torch.cat(self.parts)), 255.0)


def evaluate(gan, eval_tasks, num_averaging_runs=1, num_samples=None, batch_size=64, seed=42, num_accu_examples=204800,
             keep_features=True, real_images=None, use_graph=True, fuse_batches=4):
  """Mirrors evaluate_tfhub_module (reference eval_gan_lib.py:95-212).  Returns the result dict with
  `<label>_mean/_std/_list` keys plus `eval_samples_per_sec` (generation + Inception + statistics)."""
  dataset = gan._dataset
  n_total = num_samples or dataset.eval_test_samples
  world, rank = tpu_ops.num_replicas(), (torch.distributed.get_rank() if tpu_ops.num_replicas() > 1 else 0)
  n_local = n_total // world + (1 if rank < n_total % world else 0)
  rng = np.random.RandomState(seed + 1000 * rank)
  K.sync_stream()
  fake_dsets, timings = [], []
  n_images = max([getattr(task, "images_needed", 0) for task in eval_tasks] + [0])
  with use_ema_weights(gan):
    _update_bn_accumulators(gan, batch_size, num_accu_examples, rng)
    for _ in range(num_averaging_runs):
      acc = eval_utils.FeatureAccumulator(keep_features=keep_features)
      keeper = _ImageKeeper(n_images)
      fuse = max(1, min(int(fuse_batches), n_local // (4 * batch_size)))
      graph = _EvalBatchGraph(gan, batch_size, acc, fuse, n_images > 0) if (use_graph and n_local >= 4 * batch_size) else None
      torch.cuda.synchronize()
      t0 = time.time()
      done = 0
      if graph is not None:
        nb = n_local // (batch_size * fuse)
        graph.run_batches(rng, nb, keeper)
        done += nb * batch_size * fuse
      while done < n_local:
        imgs = generate_batch(gan, batch_size, rng)
        pool, logits = eval_utils.inception_transform(imgs)
        valid = min(batch_size, n_local - done)
        acc.add(pool, logits, valid)
        keeper.add(imgs, valid)
        done += valid
      torch.cuda.synchronize()
      timings.append(time.time() - t0)
      sample = acc.finish(eval_utils.EvalDataSample(keeper.images255()))
      if sample.activations is not None and not np.isfinite(sample.activations).all():
        raise eval_utils.NanFoundError("NaN in generated samples")
      fake_dsets.append(sample)
  if real_images is None:
    real_images = _real_images(dataset, n_total, n_local, rank, world, batch_size)
  racc = eval_utils.inception_transform_np(real_images * 255.0, batch_size, keep_features=keep_features)
  real_dset = racc.finish(eval_utils.EvalDataSample())
  result = {}
  for task in eval_tasks:
    dicts = [task.run_after_session(f, real_dset) for f in fake_dsets]
    for key in dicts[0]:
      scores = np.array([d[key] for d in dicts])
      result[key + "_mean"] = float(np.mean(scores))
      result[key + "_std"] = float(np.std(scores))
      result[key + "_list"] = "_".join(str(x) for x in scores)
  result["eval_samples_per_sec"] = n_total / float(np.mean(timings))
  if getattr(eval_utils.get_inception(), "synthetic", False):
    # scores.csv must not pass these off as comparable FID / IS values (eval_utils.get_inception)
    result["inception_weights_synthetic"] = 1.0
    if not _WARNED:
      _WARNED.append(True)
      import logging
      logging.warning("FID / IS / KID are computed with SYNTHETIC Inception weights (set $CGAN_INCEPTION_NPZ for real ones)")
  return result


_WARNED = []


def _real_images(dataset, n_total, n_local, rank, world, batch_size):
  """The real side of the metrics (reference eval_utils.get_real_images: the first num_examples of the EVAL split).  With
  a data_dir configured the images come from `dataset.eval_input_fn`, rank r taking the batches r, r+world, ...; the
  synthetic dataset draws a rank-distinct uniform sample."""
  if not getattr(dataset, "_fake_dataset", True):
    it = dataset.eval_input_fn({"batch_size": batch_size})
    out, i = [], 0
    try:
      for images, _ in it:
        if i % world == rank:
          out.append(np.array(images, np.float32, copy=True))
        it.release(1)
        i += 1
        if sum(len(o) for o in out) >= n_local:
          break
    finally:
      it.close()
    if not out:
      raise ValueError("the eval split of dataset %s is empty" % dataset.name)
    return np.concatenate(out)[:n_local]
  if world > 1:
    h, w, c = dataset.image_shape
    return np.random.RandomState(getattr(dataset, "_seed", 547) + 7919 * (rank + 1)).rand(n_local, h, w, c).astype(np.float32)
  return dataset.sample_images(n_local)
