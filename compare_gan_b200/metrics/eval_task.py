"""Abstract evaluation task (reference metrics/eval_task.py:28-76)."""
import abc


class EvalTask(object):
  """Tasks that compute a score from generated and real Inception statistics."""
  __metaclass__ = abc.ABCMeta
  _LABEL = None
  # how many generated images (the first ones of each averaging run, x255, on the device) the task reads from
  # fake_dset.images; 0: none, and the evaluation keeps no images
  images_needed = 0

  def metric_list(self):
    return frozenset(self._LABEL)

  def run_after_session(self, fake_dset, real_dset):
    """fake_dset / real_dset: eval_utils.EvalDataSample-like with .activations [N,2048] and .logits [N,1008]."""
    raise NotImplementedError()
