"""MS-SSIM sample diversity (reference metrics/ms_ssim_score.py): the mean MS-SSIM over the distinct pairs of each batch
of generated images, averaged over batches.  High values mean similar samples (mode collapse).

Deliberate differences from the reference:
  - the reference draws its batches with tf.train.shuffle_batch from the whole generated set; here they are the first
    num_batches * batch_size generated samples, in generation order.  The samples are i.i.d. draws from G, so the
    distribution is the same; which samples are scored is not pinned, the score of a given batch is;
  - with several averaging runs the reference drops the images of every run after the first (eval_gan_lib.py:179-183),
    so it could not score them; here every run keeps its first samples and is scored."""
import numpy as np

from . import eval_task
from . import image_similarity


def compute_msssim(images255, num_batches=5, batch_size=64, pair_scores=None):
  """Mean over batches of the mean MS-SSIM over the B(B-1)/2 unordered pairs of a batch of B images.  That equals the
  reference's (sum over the B^2 ordered pairs - B) / (B^2 - B) (ms_ssim_score.py:86-98): self-pairs score exactly 1 and
  MS-SSIM is symmetric.  images255: [N,h,w,c] in [0, 255] (numpy or DT).  Only whole batches are used; with fewer than
  batch_size images, one batch of all of them.  pair_scores(batch, pairs) -> [npairs] replaces the device evaluation."""
  pair_scores = pair_scores or image_similarity.pair_scores
  n = int(images255.shape[0])
  if n < 2:
    raise ValueError("MS-SSIM needs at least 2 images, got %d" % n)
  if n < batch_size:
    batch_size, num_batches = n, 1
  num_batches = min(num_batches, n // batch_size)
  pairs = np.stack(np.triu_indices(batch_size, 1), axis=1)
  scores = [np.mean(pair_scores(_rows(images255, b * batch_size, (b + 1) * batch_size), pairs)) for b in range(num_batches)]
  return float(np.mean(scores))


def _rows(images, lo, hi):
  from ..tape import DT
  return DT(images.t[lo:hi]) if isinstance(images, DT) else images[lo:hi]


class MultiscaleSSIMTask(eval_task.EvalTask):
  """MS-SSIM of the first num_batches * batch_size generated images of each averaging run.  In a sharded evaluation
  they come from rank 0's shard and the score is broadcast, so every rank returns the same value."""
  _LABEL = "ms_ssim"

  def __init__(self, num_batches=5, batch_size=64):
    self.num_batches, self.batch_size = int(num_batches), int(batch_size)
    self.images_needed = self.num_batches * self.batch_size

  def run_after_session(self, fake_dset, real_dset):
    del real_dset
    from ..tpu import tpu_ops
    if tpu_ops.num_replicas() == 1:
      return {self._LABEL: compute_msssim(fake_dset.images, self.num_batches, self.batch_size)}
    import torch
    import torch.distributed as dist
    from .. import kernels as K
    score = float("nan")
    if dist.get_rank() == 0:
      try:
        score = compute_msssim(fake_dset.images, self.num_batches, self.batch_size)
      except ValueError:
        pass            # raised on every rank below, after the broadcast
    t = torch.tensor([score], dtype=torch.float64, device=K._RT["device"])
    dist.broadcast(t, 0)
    score = float(t.item())
    if np.isnan(score):
      raise ValueError("MS-SSIM needs at least 2 generated images on rank 0")
    return {self._LABEL: score}
