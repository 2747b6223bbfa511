"""Generator conditioning (reference metrics/jacobian_conditioning.py; Odena et al. 2018, "Is Generator Conditioning
Causally Related to GAN Performance?", https://arxiv.org/abs/1802.08768): the spectrum of the metric tensor
M = J^T J of G's Jacobian J = dG(z)/dz at each latent sample, summarised by the mean and standard deviation of
log cond(M).

The Jacobian is taken in forward mode: the z_dim tangent columns of every sample are pushed through the generator's ops
in one pass (kernels.forward_mode), instead of one reverse pass per output pixel as the reference's tf.gradients loop
does (3072 per sample at CIFAR size, 49152 at 128 x 128).  M is formed on the device in float64 on the FP64 tensor cores
(csrc/jacobian.cu); the eigenvalues, condition numbers and log-determinants are numpy float64, as in the reference.

Deliberate differences from the reference:
  - the pass runs in exact fp32 (math_mode 0) whatever mode the caller uses, and restores the caller's mode afterwards:
    cond(M) = cond(J)^2, so TF32 noise of ~3e-4 in J moves log cond by order 1 once cond(J) reaches ~1e3;
  - M is accumulated in float64 from the fp32 Jacobian; the reference multiplies in float32 (np.matmul of its float32
    Jacobian), which loses the smallest eigenvalue the same way;
  - G's non-trainable state (spectral-norm u vectors, batch-norm statistics) is snapshotted before the pass, restored
    before every chunk's generator call and once more at the end, so every chunk sees the same function and the pass
    leaves G bit-identical; the reference's TF graph advances u on the one call it makes;
  - inside `evaluate`, z (and the labels of a conditional G) come from a RandomState of their own, so the FID / IS
    sample stream is the one a run without this task draws.
"""
import numpy as np

from . import eval_task

# Tangent images per chunk of the pass: every tangent of a sample is in the same chunk, so a chunk holds
# max(1, TANGENT_ROWS // z_dim) samples and the generator runs on a batch of about TANGENT_ROWS images.  This bounds the
# memory of the tangent activations to that of an inference batch of TANGENT_ROWS images.
TANGENT_ROWS = 512


def _random_state(rng):
  if rng is None:
    return np.random.mtrand._rand
  if isinstance(rng, np.random.RandomState):
    return rng
  return np.random.RandomState(rng)


def _tangent_pass(fn, x):
  """(fn(x), its tangents as a torch tensor [B, k, D]) for fn: DT [B, k] -> DT [B, ...], seeded with the identity: tangent
  j of every sample is the unit vector e_j."""
  from .. import kernels as K
  from .. import tape
  b, k = x.shape
  xt = tape.DT(x.t)
  xt.tan = K.from_numpy(np.tile(np.eye(k, dtype=np.float32), (b, 1)))
  with tape.no_record(), K.forward_mode(b, k):
    out = fn(xt)
  if out.tan is None:
    raise ValueError("the function's output does not depend on its input")
  return out, out.tan.t.reshape(b, k, -1)


def compute_jacobian(fn, xs):
  """df/dx of a batched function, [B, fx_dim, x_dim] fp32 on the device (the reference's layout): fn maps a device
  tensor (tape.DT) xs [B, x_dim] to f(xs) [B, ...], row b of the output depending on row b of xs only."""
  from .. import kernels as K
  from .. import tape
  x = xs if isinstance(xs, tape.DT) else K.from_numpy(np.asarray(xs, np.float32))
  _, t = _tangent_pass(fn, x)
  return t.transpose(1, 2).contiguous()


def _analyze_metric_tensor(metric_tensor):
  """Spectral statistics of a batch of metric tensors [batch, dim, dim], in float64: eigenvalues [batch, dim], logdet
  [batch] and log_condition_number [batch] (the 2-norm condition number, np.linalg.cond)."""
  m = np.asarray(metric_tensor, np.float64)
  eigenvalues = np.linalg.eig(m)[0]
  log_condition_number = np.log(np.linalg.cond(m))
  logdet = np.linalg.slogdet(m)[1]
  return {"eigenvalues": eigenvalues, "logdet": logdet, "log_condition_number": log_condition_number}


def analyze_metric_tensors(metric_tensors):
  """The statistics of analyze_jacobian from the metric tensors themselves ([batch, dim, dim], numpy or a device
  tensor, e.g. from kernels.metric_tensor_f64)."""
  m = metric_tensors.cpu().numpy() if hasattr(metric_tensors, "cpu") else np.asarray(metric_tensors)
  m = m.astype(np.float64)
  return {"metric_tensor": _analyze_metric_tensor(m),
          "mean_metric_tensor": _analyze_metric_tensor(m.mean(axis=0)[None])}


def analyze_jacobian(jacobian_array):
  """Statistics of the metric tensor J^T J of every Jacobian of a batch [batch, fx_dim, x_dim] and of their mean, as
  {"metric_tensor": ..., "mean_metric_tensor": ...} (see _analyze_metric_tensor)."""
  j = np.asarray(jacobian_array.cpu().numpy() if hasattr(jacobian_array, "cpu") else jacobian_array, np.float64)
  return analyze_metric_tensors(np.matmul(np.transpose(j, (0, 2, 1)), j))


def _draw_latents(gan, num_samples, rng):
  """z and labels drawn in generate_batch's order: z of the whole batch, then its labels."""
  from ..runner_lib import eval_z_generator
  z = eval_z_generator((num_samples, gan._z_dim), rng=rng)
  labels = rng.randint(0, gan._dataset.num_classes, num_samples).astype(np.int32) if gan.conditional else None
  return z, labels


class _GeneratorPass(object):
  """`with _GeneratorPass(gan) as run:` run(z, labels) -> (images DT, tangents [n, z_dim, D]) of G at those samples, in
  chunks of whole samples.  Inside the scope the library computes in exact fp32, and G's non-trainable state is restored
  before every chunk's call; on exit both are back as they were."""

  def __init__(self, gan, tangent_rows=None):
    self.gan, self.rows = gan, int(tangent_rows or TANGENT_ROWS)

  def __enter__(self):
    from .. import kernels as K
    g = self.gan
    prefix = g.generator.name + "/"
    self.state = [(v, v.t.clone()) for name, v in g.store.vars.items()
                  if name.startswith(prefix) and name not in g.store.trainable]
    self.mode = K._RT["math_mode"]
    K.set_math_mode(0)
    return self

  def _restore(self):
    for v, saved in self.state:
      v.t.copy_(saved)

  def __exit__(self, *a):
    from .. import kernels as K
    self._restore()
    K.set_math_mode(self.mode)

  def chunks(self, z, labels):
    """Yields (lo, hi, images DT, tangents [hi - lo, z_dim, D]) for consecutive chunks of the samples."""
    import torch
    from .. import kernels as K
    from .. import tape
    from .. import variables as V
    g = self.gan
    n, k = z.shape
    step = max(1, self.rows // k)
    for lo in range(0, n, step):
      hi = min(n, lo + step)
      self._restore()
      y = None
      if g.conditional:
        lab = tape.DT(torch.from_numpy(np.ascontiguousarray(labels[lo:hi])).to(K._RT["device"]))
        y = K.one_hot(lab, g._dataset.num_classes)

      def fn(zt):
        with V.use(g.store):
          return g.generator(zt, y=y, is_training=False)
      imgs, t = _tangent_pass(fn, K.from_numpy(z[lo:hi]))
      yield lo, hi, imgs, t

  def __call__(self, z, labels=None):
    import torch
    from .. import tape
    imgs, tans = [], []
    for _, _, im, t in self.chunks(z, labels):
      imgs.append(im.t)
      tans.append(t)
    return tape.DT(torch.cat(imgs)), torch.cat(tans)


def generator_metric_tensors(gan, num_samples=64, rng=None, tangent_rows=None):
  """The float64 metric tensors J^T J [num_samples, z_dim, z_dim] (numpy) of G at num_samples latent samples drawn by
  `rng` as generate_batch draws them (None: NumPy's global state)."""
  from .. import kernels as K
  z, labels = _draw_latents(gan, int(num_samples), _random_state(rng))
  parts = []
  with _GeneratorPass(gan, tangent_rows) as run:
    for _, _, _, t in run.chunks(z, labels):
      parts.append(K.metric_tensor_f64(t.contiguous()).cpu().numpy())
  return np.concatenate(parts)


def compute_generator_condition_number(gan, num_samples=64, rng=None):
  """log cond(J^T J) of G's Jacobian at each of num_samples latent samples (reference
  jacobian_conditioning.py:61-87), as a numpy float64 array."""
  m = generator_metric_tensors(gan, num_samples, rng)
  return analyze_metric_tensors(m)["metric_tensor"]["log_condition_number"]


class GeneratorConditionNumberTask(eval_task.EvalTask):
  """Count, mean and standard deviation of log cond(J^T J) over num_samples latent samples of each averaging run
  (reference jacobian_conditioning.py:32-59; 64 is the evaluation batch, eval_gan_lib.py:113).  The metric tensors
  come from `evaluate` (EvalDataSample.metric_tensors).  In a sharded evaluation rank 0 computes them and its values are
  broadcast, so every rank returns the same."""
  _CONDITION_NUMBER_COUNT = "log_condition_number_count"
  _CONDITION_NUMBER_MEAN = "log_condition_number_mean"
  _CONDITION_NUMBER_STD = "log_condition_number_std"

  def __init__(self, num_samples=64):
    self.condition_samples = int(num_samples)

  def metric_list(self):
    return frozenset([self._CONDITION_NUMBER_COUNT, self._CONDITION_NUMBER_MEAN, self._CONDITION_NUMBER_STD])

  def _score(self, fake_dset):
    m = getattr(fake_dset, "metric_tensors", None)
    if m is None:
      raise ValueError("the generator condition number needs the metric tensors of the evaluation (EvalDataSample."
                       "metric_tensors): run it through eval_gan_lib.evaluate")
    lc = analyze_metric_tensors(m)["metric_tensor"]["log_condition_number"]
    return [float(len(lc)), float(np.mean(lc)), float(np.std(lc))]

  def run_after_session(self, fake_dset, real_dset):
    del real_dset
    from ..tpu import tpu_ops
    if tpu_ops.num_replicas() == 1:
      values = self._score(fake_dset)
    else:
      import torch
      import torch.distributed as dist
      from .. import kernels as K
      values = self._score(fake_dset) if dist.get_rank() == 0 else [0.0, 0.0, 0.0]
      t = torch.tensor(values, dtype=torch.float64, device=K._RT["device"])
      dist.broadcast(t, 0)
      values = t.tolist()
    return {self._CONDITION_NUMBER_COUNT: int(values[0]), self._CONDITION_NUMBER_MEAN: values[1],
            self._CONDITION_NUMBER_STD: values[2]}
