"""Generator / discriminator base classes: the gin-facing part of a network definition.

gin files bind `G.batch_norm_fn`, `G.spectral_norm`, `D.spectral_norm`, ... (reference architectures/abstract_arch.py:
48-146); a concrete network only supplies `apply`.  Calling the object opens the network's variable scope
("generator" / "discriminator" — the root of the checkpoint key space) and runs the definition.
"""
from .. import gin_lite as gin
from .. import kernels as K
from .. import tape
from .. import utils
from .. import variables as V


class _Network(object):
  """What generators and discriminators share: a named variable scope and the configured normalisation."""

  # cut a recomputed segment (tape.segment) per residual / non-local block; set by ModularGAN.build when the activation
  # stash of a training update would not fit in device memory
  recompute = False

  def _setup(self, name, batch_norm_fn, spectral_norm):
    self._name = name
    self._batch_norm_fn = batch_norm_fn
    self._spectral_norm = spectral_norm

  name = property(lambda self: self._name)

  @property
  def trainable_variables(self):
    return list(V.current().trainable_under(self._name).values())

  def _run(self, **inputs):
    # one batched spectral-norm launch per call for the network's small weights (kernels.SNBatch), keyed by the variable
    # store in use (a network object may be run against several stores in tests)
    states = self.__dict__.setdefault("_sn_states", {})
    store = V.current()
    state = states.get(id(store))
    if state is None or state[0]() is not store:
      import weakref
      state = states[id(store)] = (weakref.ref(store), K.SNBatch())
    with K.sn_batch(state[1]), V.variable_scope(self._name), tape.segments(self.recompute):
      return self.apply(**inputs)

  def batch_norm(self, inputs, **kwargs):
    """Applies the configured batch-norm function with whichever of (z, y, is_training, name, use_sn, ...) it accepts;
    the identity when none is configured (reference abstract_arch.py:76-83, 121-128)."""
    if self._batch_norm_fn is None:
      return inputs
    kwargs.setdefault("use_sn", self._spectral_norm)
    return utils.call_with_accepted_args(self._batch_norm_fn, inputs=inputs, **kwargs)


@gin.configurable("G", blacklist=["name", "image_shape"])
class AbstractGenerator(_Network):
  """z (and one-hot y) -> images in [0, 1]."""

  def __init__(self, name="generator", image_shape=None, batch_norm_fn=None, spectral_norm=False):
    self._setup(name, batch_norm_fn, spectral_norm)
    self._image_shape = image_shape

  def __call__(self, z, y, is_training, reuse=None):
    return self._run(z=z, y=y, is_training=is_training)

  def apply(self, z, y, is_training):
    raise NotImplementedError


@gin.configurable("D", blacklist=["name"])
class AbstractDiscriminator(_Network):
  """images (and one-hot y) -> (probability, logit, penultimate features)."""

  def __init__(self, name="discriminator", batch_norm_fn=None, layer_norm=False, spectral_norm=False):
    # read by the residual-block discriminators (resnet_ops / resnet_biggan); the others ignore it, as the reference's do
    self._setup(name, batch_norm_fn, spectral_norm)
    self._layer_norm = layer_norm

  def __call__(self, x, y, is_training, reuse=None):
    return self._run(x=x, y=y, is_training=is_training)

  def apply(self, x, y, is_training):
    raise NotImplementedError
