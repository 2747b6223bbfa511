"""Ops library: same names, arguments and error behaviour as the reference's
compare_gan/architectures/arch_ops.py, with every computation dispatched to sm_90a kernels
through the C-ABI (kernels.py).  Inputs/outputs are device tensors (tape.DT), NHWC float32.
"""
import functools

import numpy as np

from .. import gin_lite as gin
from .. import kernels as K
from .. import tape
from .. import variables as V
from ..gans import consts
from ..tpu import tpu_ops


# test hook: callables fn(scope_name, tensor) receiving the output of every linear / un-fused conv2d / deconv2d /
# non_local_block / residual block, keyed by the variable scope it ran in (the oracle has the same hook); once per forward,
# not again when a recomputed segment replays it
ACT_OBSERVERS = []


def observe(y, suffix=None):
  if ACT_OBSERVERS and not tape.replaying():
    name = "/".join(V.current()._scope + ([suffix] if suffix else []))
    for fn in ACT_OBSERVERS:
      fn(name, y)
  return y


def recomputed(fn, *inputs):
  """fn(*inputs) as one recomputed segment of the tape (tape.segment; a residual or non-local block, when the network
  recomputes its blocks): its backward replays fn in the variable store and scope of the first pass."""
  store = V.current()
  scope = list(store._scope)

  def run(*xs):
    with V.use(store), store.at_scope(scope):
      return fn(*xs)
  return tape.segment(run, list(inputs))


# ----------------------------------------------------------------------------- initializers

def _normal(stddev):
  return lambda rng, shape: rng.standard_normal(shape) * stddev


def _truncated_normal(stddev):
  def init(rng, shape):
    a = rng.standard_normal(shape)
    bad = np.abs(a) > 2.0
    while bad.any():
      a[bad] = rng.standard_normal(int(bad.sum()))
      bad = np.abs(a) > 2.0
    return a * stddev
  return init


def _orthogonal(rng, shape):
  rows, cols = int(np.prod(shape[:-1])), int(shape[-1])
  a = rng.standard_normal((max(rows, cols), min(rows, cols)))
  q, r = np.linalg.qr(a)
  q = q * np.sign(np.diag(r))
  if rows < cols:
    q = q.T
  return q.reshape(shape)


def glorot_normal(rng, shape):
  """tf.initializers.glorot_normal (resnet_biggan.py:415-417)."""
  std = np.sqrt(2.0 / (shape[0] + shape[1])) / .87962566103423978
  return _truncated_normal(std)(rng, shape)


def zeros_init(rng, shape):
  return np.zeros(shape, np.float32)


def ones_init(rng, shape):
  return np.ones(shape, np.float32)


def constant_init(v):
  return lambda rng, shape: np.full(shape, v, np.float32)


@gin.configurable("weights")
def weight_initializer(initializer=consts.NORMAL_INIT, stddev=0.02):
  """Returns the initializer for the given name (reference arch_ops.py:46-63)."""
  if initializer == consts.NORMAL_INIT:
    return _normal(stddev)
  if initializer == consts.TRUNCATED_INIT:
    return _truncated_normal(stddev)
  if initializer == consts.ORTHOGONAL_INIT:
    return _orthogonal
  raise ValueError("Unknown weight initializer {}.".format(initializer))


# ----------------------------------------------------------------------------- batch norm

def _bn_state(c, use_moving_averages):
  """Creates/fetches the non-trainable BN variables in the current scope (arch_ops.py:66-191)."""
  st = K.BNState()
  if use_moving_averages:
    st.moving_mean = V.get_variable("moving_mean", (c,), zeros_init, trainable=False)
    st.moving_var = V.get_variable("moving_variance", (c,), ones_init, trainable=False)
  else:
    with V.variable_scope("accu"):
      st.accu_mean = V.get_variable("accu_mean", (c,), zeros_init, trainable=False)
      st.accu_var = V.get_variable("accu_variance", (c,), zeros_init, trainable=False)
      st.accu_counter = V.get_variable("accu_counter", (), constant_init(1e-12), trainable=False)
      st.update_accus = V.get_variable("update_accus", (), zeros_init, trainable=False)
  return st


@gin.configurable(whitelist=["decay", "epsilon", "use_cross_replica_mean", "use_moving_averages"])
def standardize_batch(inputs, is_training, decay=0.999, epsilon=1e-3, data_format="NHWC",
                      use_moving_averages=True, use_cross_replica_mean=None,
                      _gamma=None, _beta=None, _cond=False, _relu=False, _tf32=False, _gamma_beta=None):
  """Batch standardisation (reference arch_ops.py:194-319).  The private `_gamma/_beta` arguments let
  batch_norm / conditional_batch_norm fuse their scale+offset (and a following ReLU) into the same kernel
  (`_gamma_beta`: self_modulated_batch_norm's [2N, C] scale and offset); `_tf32` says that the result only feeds
  tensor-core contractions (it is then stored TF32-rounded in math_mode 1)."""
  if data_format not in {"NCHW", "NHWC"}:
    raise ValueError("Invalid data_format {}. Allowed: NCHW, NHWC.".format(data_format))
  if data_format != "NHWC":
    raise ValueError("Only NHWC is implemented on the H100 path.")
  if use_cross_replica_mean is None:
    use_cross_replica_mean = tpu_ops.num_replicas() > 1
  rank = len(inputs.shape)
  if rank not in (2, 4):
    raise ValueError("Inputs has unsupported rank. Expected 2 or 4 but got %d" % rank)
  c = inputs.shape[-1]
  st = _bn_state(c, use_moving_averages)
  extra = {} if _gamma_beta is None else {"gamma_beta": _gamma_beta}
  if is_training:
    return K.bn_train(inputs, _gamma, _beta, epsilon, st if use_moving_averages else None, decay, cond=_cond,
                      relu_after=_relu, allreduce=tpu_ops.cross_replica_sum_ if use_cross_replica_mean else None,
                      world=tpu_ops.num_replicas() if use_cross_replica_mean else 1, round_out=_tf32, **extra)
  return K.bn_infer(inputs, _gamma, _beta, epsilon, st, use_moving_averages, cond=_cond, relu_after=_relu,
                    round_out=_tf32, **extra)


@gin.configurable(blacklist=["inputs"])
def no_batch_norm(inputs):
  return inputs


@gin.configurable(blacklist=["inputs", "is_training", "center", "scale", "name"])
def batch_norm(inputs, is_training, center=True, scale=True, name="batch_norm", _relu=False, _tf32=False):
  """Vanilla batch norm with trainable gamma/beta (reference arch_ops.py:327-367)."""
  with V.variable_scope(name):
    c = inputs.shape[-1]
    # variable creation order as in the reference: moving stats, then gamma, beta
    _bn_state_peek(c)
    gamma = V.get_variable("gamma", (c,), ones_init) if scale else None
    beta = V.get_variable("beta", (c,), zeros_init) if center else None
    return standardize_batch(inputs, is_training=is_training, _gamma=gamma, _beta=beta, _relu=_relu, _tf32=_tf32)


def _bn_state_peek(c):
  """Create the BN state variables first so that variable order matches the reference graph."""
  cfg = gin._bound_kwargs("arch_ops.standardize_batch")
  _bn_state(c, bool(cfg.get("use_moving_averages", True)))


@gin.configurable(whitelist=["use_bias"])
def conditional_batch_norm(inputs, y, is_training, use_sn, center=True, scale=True, name="batch_norm",
                           use_bias=False, _relu=False, _tf32=False):
  """Conditional batch normalization (reference arch_ops.py:423-445): gamma(y), beta(y) = linear(y)."""
  if y is None:
    raise ValueError("You must provide y for conditional batch normalization.")
  if len(y.shape) != 2:
    raise ValueError("Conditioning must have rank 2.")
  with V.variable_scope(name):
    c = inputs.shape[-1]
    _bn_state_peek(c)
    gamma = beta = None
    with V.variable_scope("condition"):
      if scale:
        gamma = linear(y, c, scope="gamma", use_sn=use_sn, use_bias=use_bias)
      if center:
        beta = linear(y, c, scope="beta", use_sn=use_sn, use_bias=use_bias)
    return standardize_batch(inputs, is_training=is_training, _gamma=gamma, _beta=beta, _cond=True, _relu=_relu,
                             _tf32=_tf32)


@gin.configurable(whitelist=["num_hidden"])
def self_modulated_batch_norm(inputs, z, is_training, use_sn, center=True, scale=True, name="batch_norm",
                              num_hidden=32, _relu=False, _tf32=False):
  """Self-modulated batch norm (reference arch_ops.py:370-420; Chen et al. 2019): gamma and beta are an MLP of z,
  gamma = linear(h) with bias 1, beta = linear(h), h = relu(linear(z, num_hidden)) or z itself when num_hidden = 0.
  The MLP is one kernel (kernels.self_modulation); its [2N, C] output feeds the BN apply as a conditional gamma / beta."""
  if z is None:
    raise ValueError("You must provide z for self modulation.")
  if not (center and scale):
    raise NotImplementedError("self_modulated_batch_norm without its scale or offset is not implemented")
  with V.variable_scope(name):
    c = inputs.shape[-1]
    _bn_state_peek(c)
    with V.variable_scope("sbn"):
      wh = bh = None
      if num_hidden > 0:
        with V.variable_scope("hidden"):
          wh, bh = _linear_params(z.shape[1], num_hidden, use_sn=use_sn)
      width = num_hidden if num_hidden > 0 else z.shape[1]
      with V.variable_scope("gamma"):
        wg, bg = _linear_params(width, c, bias_start=1.0, use_sn=use_sn)
      with V.variable_scope("beta"):
        wb, bb = _linear_params(width, c, use_sn=use_sn)
      gamma_beta = K.self_modulation(z, wh, bh, wg, bg, wb, bb)
    return standardize_batch(inputs, is_training=is_training, _gamma_beta=gamma_beta, _cond=True, _relu=_relu,
                             _tf32=_tf32)


def _linear_params(input_size, output_size, bias_start=0.0, use_sn=False):
  """(kernel, bias) of a `linear` layer in the current scope, created as linear creates them: kernel, its u_var under
  use_sn, bias."""
  kernel = V.get_variable("kernel", (input_size, output_size), weight_initializer(stddev=0.02))
  if use_sn:
    kernel = spectral_norm(kernel)
  return kernel, V.get_variable("bias", (output_size,), constant_init(bias_start))


def configured_norm(norm_fn):
  """The gin-configured normaliser behind a network's `batch_norm` method (None when it is the identity)."""
  net = getattr(norm_fn, "__self__", None)
  fn = getattr(net, "_batch_norm_fn", None) if net is not None else None
  return None if fn is no_batch_norm else fn


def norm_relu(norm_fn, inputs, _tf32=False, **kwargs):
  """relu(norm_fn(inputs)): when the configured normaliser is one of the BN kernels above, the ReLU is fused into the
  BN-apply kernel (one pass over the activation instead of two); any other normaliser is followed by a plain ReLU.
  `_tf32`: the result only feeds tensor-core contractions (stored TF32-rounded in math_mode 1)."""
  if configured_norm(norm_fn) in (batch_norm, conditional_batch_norm, self_modulated_batch_norm):
    return norm_fn(inputs, _relu=True, _tf32=_tf32, **kwargs)
  return K.relu(norm_fn(inputs, **kwargs), round_tf32=_tf32)


def layer_norm(inputs, is_training, scope, _relu=False, _tf32=False):
  """tf.contrib.layers.layer_norm(inputs, trainable=is_training, scope=scope) (reference arch_ops.py:448-450): moments
  per sample over H, W and C, beta / gamma per channel (created in that order, zeros / ones).  `_relu` fuses the
  following ReLU, `_tf32` as in norm_relu."""
  with V.variable_scope(scope):
    c = inputs.shape[-1]
    beta = V.get_variable("beta", (c,), zeros_init, trainable=is_training)
    gamma = V.get_variable("gamma", (c,), ones_init, trainable=is_training)
  return K.layer_norm(inputs, gamma, beta, relu_after=_relu, round_out=_tf32)


# ----------------------------------------------------------------------------- spectral norm

@gin.configurable(blacklist=["inputs"])
def spectral_norm(inputs, epsilon=1e-12, singular_value="left", _var_name="kernel"):
  """Spectral normalisation of a weight tensor (reference arch_ops.py:453-535)."""
  if len(inputs.shape) < 2:
    raise ValueError("Spectral norm can only be applied to multi-dimensional tensors")
  rows = int(np.prod(inputs.shape[:-1]))
  cols = inputs.shape[-1]
  if singular_value == "auto":
    singular_value = "left" if rows <= cols else "right"
  left = singular_value == "left"
  u_shape = (rows, 1) if left else (1, cols)
  u_var = V.get_variable(_var_name + "/u_var", u_shape, _normal(1.0), trainable=False)
  return K.spectral_normalize(inputs, u_var, left, epsilon)


# ----------------------------------------------------------------------------- layers

def linear(inputs, output_size, scope=None, stddev=0.02, bias_start=0.0, use_sn=False, use_bias=True):
  """Linear layer without the non-linear activation applied (reference arch_ops.py:538-556)."""
  shape = inputs.shape
  with V.variable_scope(scope or "linear"):
    kernel = V.get_variable("kernel", (shape[1], output_size), weight_initializer(stddev=stddev))
    if use_sn:
      kernel = spectral_norm(kernel)
    outputs = K.matmul(inputs, kernel)
    if use_bias:
      bias = V.get_variable("bias", (output_size,), constant_init(bias_start))
      outputs = K.bias_add(outputs, bias)
    return observe(outputs)


def conv2d(inputs, output_dim, k_h, k_w, d_h, d_w, stddev=0.02, name="conv2d", use_sn=False, use_bias=True,
           _upsample=False, _relu=False, _residual=None, _tf32=False):
  """2-D convolution, SAME padding (reference arch_ops.py:559-573).  `_upsample` fuses the preceding
  resnet_ops.unpool; `_residual` / `_relu` / `_tf32` are the epilogue fusions of kernels.conv2d."""
  if d_h != d_w:
    raise ValueError("Only square strides are supported.")
  with V.variable_scope(name):
    w = V.get_variable("kernel", (k_h, k_w, inputs.shape[-1], output_dim), weight_initializer(stddev=stddev))
    if use_sn:
      w = spectral_norm(w)
    bias = V.get_variable("bias", (output_dim,), zeros_init) if use_bias else None
    y = K.conv2d(inputs, w, bias, stride=d_h, upsample=_upsample, relu=_relu, residual=_residual, round_out=_tf32)
    return y if (_relu or _residual is not None) else observe(y)


conv1x1 = functools.partial(conv2d, k_h=1, k_w=1, d_h=1, d_w=1)


def deconv2d(inputs, output_shape, k_h, k_w, d_h, d_w, stddev=0.02, name="deconv2d", use_sn=False):
  """Transposed 2-D convolution (reference arch_ops.py:579-592)."""
  with V.variable_scope(name):
    w = V.get_variable("kernel", (k_h, k_w, output_shape[-1], inputs.shape[-1]),
                       weight_initializer(stddev=stddev))
    if use_sn:
      w = spectral_norm(w)
    bias = V.get_variable("bias", (output_shape[-1],), zeros_init)
    return observe(K.deconv2d(inputs, w, bias, (output_shape[1], output_shape[2]), d_h))


def lrelu(inputs, leak=0.2, name="lrelu", _tf32=False):
  """Leaky ReLU max(x, leak*x) (reference arch_ops.py:595-597)."""
  return K.lrelu(inputs, leak, round_tf32=_tf32)


def non_local_block(x, name, use_sn):
  """Self-attention (non-local) block (reference arch_ops.py:709-758); one recomputed segment."""
  return recomputed(lambda x_: _non_local_block(x_, name, use_sn), x)


def _non_local_block(x, name, use_sn):
  with V.variable_scope(name):
    n, h, w, num_channels = x.shape
    num_channels_attn = num_channels // 8
    num_channels_g = num_channels // 2
    # the fused attention kernel reads theta / phi / g as TF32 operands: their producers store them rounded
    fused = K.attention_shape_ok(n, h * w, h * w // 4, num_channels_attn, num_channels_g)
    theta = conv1x1(x, num_channels_attn, name="conv2d_theta", use_sn=use_sn, use_bias=False, _tf32=fused)
    theta = K.reshape(theta, n, h * w, num_channels_attn)
    phi = conv1x1(x, num_channels_attn, name="conv2d_phi", use_sn=use_sn, use_bias=False, _tf32=fused)
    phi = K.maxpool2(phi)
    phi = K.reshape(phi, n, h * w // 4, num_channels_attn)
    g = conv1x1(x, num_channels_g, name="conv2d_g", use_sn=use_sn, use_bias=False, _tf32=fused)
    g = K.maxpool2(g)
    g = K.reshape(g, n, h * w // 4, num_channels_g)
    # attn = softmax(theta phi^T); attn_g = attn g (arch_ops.py:744-753): one fused kernel where the shape allows
    attn_g = K.attention(theta, phi, g)
    attn_g = K.reshape(attn_g, n, h, w, num_channels_g)
    sigma = V.get_variable("sigma", (), zeros_init)
    attn_g = conv1x1(attn_g, num_channels, name="conv2d_attn_g", use_sn=use_sn, use_bias=False)
    return observe(K.add(x, K.scale_by_param(attn_g, sigma)))
