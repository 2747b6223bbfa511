"""Abstract evaluation task (reference metrics/eval_task.py:28-76)."""
import abc


class EvalTask(object):
  """Tasks that compute a score from generated and real Inception statistics."""
  __metaclass__ = abc.ABCMeta
  _LABEL = None
  # how many generated images (the first ones of each averaging run, x255, on the device) the task reads from
  # fake_dset.images; 0: none, and the evaluation keeps no images
  images_needed = 0
  # how many seed samples (the first ones of each averaging run) the task needs the float64 distances of every generated
  # sample to, in fake_dset.seed_distances [n, seeds]; 0: none, and the evaluation measures none
  distance_seeds = 0
  # how many latent samples the task needs the float64 metric tensors J^T J of G's Jacobian at, in
  # fake_dset.metric_tensors [n, z_dim, z_dim]; 0: none, and the evaluation computes none
  condition_samples = 0

  def metric_list(self):
    return frozenset(self._LABEL)

  def run_after_session(self, fake_dset, real_dset):
    """fake_dset / real_dset: eval_utils.EvalDataSample-like with .activations [N,2048] and .logits [N,1008]."""
    raise NotImplementedError()
