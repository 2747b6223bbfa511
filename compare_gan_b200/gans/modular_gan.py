"""ModularGAN: the training step (reference gans/modular_gan.py:56-670) on one H100 per process.

What TF did with a static graph + TPUEstimator is done here with:
  * an eager "cycle" (disc_iters D-updates + 1 G-update, the unrolled/TPU semantics of
    model_fn :512-604) written against the taped C-ABI ops, and
  * CUDA-graph capture of that whole cycle (streams + graphs instead of a tracing compiler), so the
    per-step host cost is one graph launch; all state (weights, Adam moments, BN moving averages,
    spectral-norm u vectors, step counters, EMA shadows) lives in HBM and is updated in place.
Data parallelism: one process per GPU, gradients of a flat per-network buffer are all-reduced
with NCCL (CrossShardOptimizer, :606-616) and BN moments are all-reduced inside standardize_batch.
"""
import numpy as np
import torch

from .. import gin_lite as gin
from .. import kernels as K
from .. import tape
from .. import variables as V
from ..architectures import (dcgan, infogan, resnet5, resnet30, resnet_biggan, resnet_biggan_deep, resnet_cifar,
                             resnet_stl, sndcgan)
from ..tpu import tpu_ops
from . import consts, loss_lib, penalty_lib
from .abstract_gan import AbstractGAN


class AdamOptimizer(object):
  """tf.train.AdamOptimizer hyper-parameters; the update itself is cgan_adam_step (TF form:
  lr_t = lr*sqrt(1-b2^t)/(1-b1^t), eps outside the corrected sqrt)."""

  def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8):
    self.learning_rate, self.beta1, self.beta2, self.epsilon = learning_rate, beta1, beta2, epsilon


gin.external_configurable(AdamOptimizer, "tf.train.AdamOptimizer")


HEADROOM_BYTES = 12 << 30


def memory_budget():
  """Device bytes the activation stash of a training update may take: what the device and torch's allocator cache hold
  free when the model is built, less HEADROOM_BYTES for the backward pass's working tensors (a recomputed block's replay
  among them) and the allocator's fragmentation.  None without a CUDA device (the CPU emulator of the C-ABI).  Tests
  replace this function to force recomputation."""
  if K._RT["device"].type != "cuda":
    return None
  free, _ = torch.cuda.mem_get_info()
  return free + torch.cuda.memory_reserved() - torch.cuda.memory_allocated() - HEADROOM_BYTES


class _FlatAdam(object):
  def __init__(self, opt, flat):
    self.opt, self.flat = opt, flat
    n = flat["total"]
    dev = flat["param"].t.device
    self.m = tape.DT(torch.zeros(n, dtype=torch.float32, device=dev))
    self.v = tape.DT(torch.zeros(n, dtype=torch.float32, device=dev))
    self.step = torch.zeros(1, dtype=torch.int32, device=dev)

  def apply(self, grad_scale, ema=None, ema_decay=0.0, ema_start=0):
    o, f = self.opt, self.flat
    K._call("adam_step", f["param"].ptr, f["grad"].ptr, self.m.ptr, self.v.ptr, f["total"], float(o.learning_rate),
            float(o.beta1), float(o.beta2), float(o.epsilon), float(grad_scale), self.step.data_ptr(),
            None if ema is None else ema.ptr, float(ema_decay), int(ema_start))


@gin.configurable(blacklist=["dataset", "parameters", "model_dir"])
class ModularGAN(AbstractGAN):
  """Gin-configurable GAN (reference gans/modular_gan.py:56-165 constructor contract)."""

  def __init__(self, dataset, parameters, model_dir, deprecated_split_disc_calls=False,
               experimental_joint_gen_for_disc=False, experimental_force_graph_unroll=False, g_use_ema=False,
               ema_decay=0.9999, ema_start_step=40000, g_optimizer_fn=AdamOptimizer, d_optimizer_fn=None,
               g_lr=0.0002, d_lr=None, conditional=False, fit_label_distribution=False, math_mode=0):
    super(ModularGAN, self).__init__(dataset=dataset, parameters=parameters, model_dir=model_dir)
    if deprecated_split_disc_calls or fit_label_distribution or experimental_joint_gen_for_disc:
      raise NotImplementedError("deprecated_split_disc_calls / fit_label_distribution / experimental_joint_gen_for_disc are "
                                "outside the hot path (the last one changes G's batch statistics and must not be ignored)")
    self._experimental_joint_gen_for_disc = experimental_joint_gen_for_disc
    self._g_use_ema = g_use_ema
    self._ema_decay = ema_decay
    self._ema_start_step = ema_start_step
    self._g_optimizer_fn = g_optimizer_fn
    self._d_optimizer_fn = d_optimizer_fn if d_optimizer_fn is not None else g_optimizer_fn
    self._g_lr = g_lr
    self._d_lr = g_lr if d_lr is None else d_lr
    if conditional and not self._dataset.num_classes:
      raise ValueError("Option 'conditional' selected but dataset {} does not have labels".format(
          self._dataset.name))
    self._conditional = conditional
    # 0: exact fp32 contractions (parity mode); 1: wgmma TF32 tensor-core convolutions (RN-rounded operands)
    self._math_mode = math_mode
    self._architecture = parameters["architecture"]
    self._z_dim = parameters["z_dim"]
    self._lambda = parameters["lambda"]
    self._disc_iters = parameters.get("disc_iters", 1)
    self.d_loss = None
    self.g_loss = None
    self.penalty_loss = None
    self._discriminator = None
    self._generator = None
    self.store = V.VariableStore(seed=parameters.get("seed", 0))
    self._graph = None
    self._built_batch = None
    self.d_kernels = None            # K.KernelSegments of D's kernels when the bound penalty is l2_penalty
    self.recompute = {"generator": False, "discriminator": False}     # per network: blocks recomputed (see build)

  # ---- architecture registry (reference :169-213) ---------------------------------------------
  @property
  def conditional(self):
    return self._conditional

  @property
  def generator(self):
    if self._generator is None:
      module = {consts.RESNET5_ARCH: resnet5, consts.RESNET_BIGGAN_ARCH: resnet_biggan, consts.DCGAN_ARCH: dcgan,
                consts.RESNET_BIGGAN_DEEP_ARCH: resnet_biggan_deep,
                consts.RESNET_CIFAR_ARCH: resnet_cifar, consts.SNDCGAN_ARCH: sndcgan, consts.RESNET30_ARCH: resnet30,
                consts.RESNET_STL_ARCH: resnet_stl, consts.INFOGAN_ARCH: infogan}.get(self._architecture)
      if module is None:
        raise NotImplementedError("Architecture {} not implemented.".format(self._architecture))
      self._generator = module.Generator(image_shape=self._dataset.image_shape)
    return self._generator

  @property
  def discriminator(self):
    if self._discriminator is None:
      module = {consts.RESNET5_ARCH: resnet5, consts.RESNET_BIGGAN_ARCH: resnet_biggan, consts.DCGAN_ARCH: dcgan,
                consts.RESNET_BIGGAN_DEEP_ARCH: resnet_biggan_deep,
                consts.RESNET_CIFAR_ARCH: resnet_cifar, consts.SNDCGAN_ARCH: sndcgan, consts.RESNET30_ARCH: resnet30,
                consts.RESNET_STL_ARCH: resnet_stl, consts.INFOGAN_ARCH: infogan}.get(self._architecture)
      if module is None:
        raise NotImplementedError("Architecture {} not implemented.".format(self._architecture))
      self._discriminator = module.Discriminator()
    return self._discriminator

  def _get_one_hot_labels(self, labels):
    """reference :359-363."""
    if not self.conditional:
      raise ValueError("_get_one_hot_labels() called but GAN is not conditional.")
    return K.one_hot(labels, self._dataset.num_classes)

  # ---- loss (reference create_loss :618-670) ------------------------------------------------------
  def create_loss(self, features, labels, params=None, is_training=True, for_discriminator=True):
    """Sets self.d_loss / self.g_loss.  features: dict with "images", "generated" (+"sampled_labels", "alpha").
    As in TF, the penalty sub-graph only runs when d_loss is the fetched tensor."""
    images = features["images"]
    generated = features["generated"]
    if self.conditional:
      y = self._get_one_hot_labels(labels)
      sampled_y = self._get_one_hot_labels(features["sampled_labels"])
      all_y = K.concat_rows(y, sampled_y)
    else:
      y = sampled_y = all_y = None
    all_images = K.concat_rows(images, generated)
    d_all, d_all_logits, _ = self.discriminator(all_images, y=all_y, is_training=is_training)
    b = images.shape[0]
    d_real, d_fake = K.slice_rows(d_all, 0, b), K.slice_rows(d_all, b, 2 * b)
    d_real_logits, d_fake_logits = K.slice_rows(d_all_logits, 0, b), K.slice_rows(d_all_logits, b, 2 * b)
    self.d_loss, _, _, self.g_loss = loss_lib.get_losses(
        d_real=d_real, d_fake=d_fake, d_real_logits=d_real_logits, d_fake_logits=d_fake_logits)
    if for_discriminator:
      penalty_loss = penalty_lib.get_penalty_loss(
          x=images, x_fake=generated, y=y, is_training=is_training, discriminator=self.discriminator,
          alpha=features.get("alpha"), step=self.d_opt.step, kernel_segments=self.d_kernels)
      self.penalty_loss = penalty_loss
      if penalty_loss.node is not None:
        self.d_loss = K.add(self.d_loss, K.affine(penalty_loss, self._lambda))

  # ---- build -----------------------------------------------------------------------------------------
  def build(self, batch_size):
    """Creates all variables (one dry G/D call, like TF graph construction), packs them into flat buffers,
    creates optimizer state and the static input buffers for `batch_size` per sub-step."""
    K.lib()
    K.sync_stream()
    K.set_math_mode(self._math_mode)
    k = self._disc_iters
    h, w, c = self._dataset.image_shape
    dev = K._RT["device"]
    b = batch_size
    self.inputs = []
    for _ in range(k + 1):
      f = {"images": tape.DT(torch.zeros(b, h, w, c, device=dev)), "z": tape.DT(torch.zeros(b, self._z_dim, device=dev))}
      if self.conditional:
        f["labels"] = tape.DT(torch.zeros(b, dtype=torch.int32, device=dev))
        f["sampled_labels"] = tape.DT(torch.zeros(b, dtype=torch.int32, device=dev))
      f["alpha"] = tape.DT(torch.zeros(b, 1, 1, 1, device=dev))
      self.inputs.append(f)
    self.losses = tape.DT(torch.zeros(k + 1, device=dev))
    with V.use(self.store), tape.no_record():
      self._build_networks(self.inputs[0])
    self.flat_g = self.store.pack("generator")
    self.flat_d = self.store.pack("discriminator")
    self.store.reset_to_init()          # graph construction runs no ops: undo BN/u_var side effects
    self.g_opt = _FlatAdam(self._g_optimizer_fn(self._g_lr), self.flat_g)
    self.d_opt = _FlatAdam(self._d_optimizer_fn(self._d_lr), self.flat_d)
    if penalty_lib.bound_penalty() is penalty_lib.l2_penalty:
      self.d_kernels = K.KernelSegments(self.flat_d, penalty_lib.l2_kernels(self.store.trainable_under("discriminator")))
    self.ema = None
    if self._g_use_ema:
      self.ema = tape.DT(self.flat_g["param"].t.clone())
    self.recompute = self._choose_recompute(b)
    self.generator.recompute = self.recompute["generator"]
    self.discriminator.recompute = self.recompute["discriminator"]
    self._built_batch = b
    torch.cuda.synchronize()
    return self

  def _choose_recompute(self, b):
    """Which networks recompute their blocks in the backward pass (tape.segment) instead of stashing their activations.
    The stash of each network, plain and segmented, is measured after one recorded forward at 1 and at 2 images per
    replica and extrapolated linearly to the built batch (B images for G, 2B for D); a D-update holds D's stash, a
    G-update G's and D's.  The first choice among: nothing, the network with the larger stash, both, whose two updates
    fit memory_budget() is taken.  A second-order gradient penalty differentiates through D twice, which a replay does
    not support: such a model keeps the stash path, as does any model off the GPU unless the budget is forced."""
    none = {"generator": False, "discriminator": False}
    budget = memory_budget()
    if budget is None or penalty_lib.bound_penalty() in (penalty_lib.wgangp_penalty, penalty_lib.dragan_penalty):
      return none
    at1, at2 = self._stash_bytes(1), self._stash_bytes(2)
    self.store.reset_to_init()           # undo the measurement's BN / u_var updates
    stash = {k: at1[k] + (at2[k] - at1[k]) * ((2 * b if k[0] == "discriminator" else b) - 1) for k in at1}
    self.predicted_stash = dict(stash, budget=budget)          # (read by profiles/prof_biggan_batch256.py)

    def fits(choice):
      g, d = stash[("generator", choice["generator"])], stash[("discriminator", choice["discriminator"])]
      return max(d, g + d) <= budget
    larger = max(("generator", "discriminator"), key=lambda n: stash[(n, False)] - stash[(n, True)])
    for choice in (none, dict(none, **{larger: True})):
      if fits(choice):
        return choice
    return {"generator": True, "discriminator": True}

  def _stash_bytes(self, n):
    """{(network, segmented): device bytes one recorded forward at n images per replica keeps alive} (0 off the GPU)."""
    out = {}
    cuda = K._RT["device"].type == "cuda"
    h, w, c = self._dataset.image_shape
    dev = K._RT["device"]
    z = tape.DT(torch.zeros(n, self._z_dim, device=dev))
    images = tape.DT(torch.zeros(n, h, w, c, device=dev))
    labels = tape.DT(torch.zeros(n, dtype=torch.int32, device=dev))
    for name, net, x in (("generator", self.generator, z), ("discriminator", self.discriminator, images)):
      for seg in (False, True):
        out[(name, seg)] = 0
        if not cuda:
          continue
        net.recompute = seg
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        with V.use(self.store), tape.record(True):
          y = self._get_one_hot_labels(labels) if self.conditional else None
          held = net(x, y=y, is_training=True)
          torch.cuda.synchronize()
          out[(name, seg)] = torch.cuda.memory_allocated() - before
        del held, y
        net.recompute = False
    return out

  def _build_networks(self, f):
    """One dry generator / discriminator call that creates every variable (like TF graph construction)."""
    sy = self._get_one_hot_labels(f["sampled_labels"]) if self.conditional else None
    gen = self.generator(f["z"], y=sy, is_training=True)
    all_y = K.concat_rows(sy, sy) if self.conditional else None
    self.discriminator(K.concat_rows(f["images"], gen), y=all_y, is_training=True)
    return gen, all_y

  # ---- one cycle (reference model_fn :512-604, unrolled) -------------------------------------------------
  def _grad_sinks(self, prefix, params):
    """{id(variable): its slot in the flat gradient buffer}: tape.backward lets the vjp that produces a variable's
    gradient write it there directly (kernels._grad_out)."""
    return {id(v): self.store.grad_view(prefix, name) for name, v in params.items()}

  def _apply_grads(self, prefix, flat, grads, names):
    for name, g in zip(names, grads):
      view = self.store.grad_view(prefix, name)
      if g is None:
        K.fill_(view, 0.0)                      # unreachable variable: zero gradient (tf.gradients would return None)
      elif g.ptr != view.ptr:                   # accumulated from several uses, or produced by an op without a sink
        K.copy_(view, g)
    if prefix == "discriminator" and self.d_kernels is not None:
      self.d_kernels.add_pending_grads()        # the L2 penalty's term, identical on every replica: the mean keeps it
    world = tpu_ops.num_replicas()
    if world > 1:
      tpu_ops.cross_replica_sum_(flat["grad"])
    return 1.0 / world

  def _cycle(self):
    k = self._disc_iters
    with V.use(self.store):
      # _split_inputs_and_generate_samples (:428-469).  G's weights only change in the last sub-step, so the sample each
      # D-update consumes is generated right before that update and freed after it, and the differentiated sample of
      # the G-update is generated after the D-updates: same values as generating all k+1 up front (the TF graph leaves
      # the order of the BN moving-average update ops undefined), but the G activation stash no longer lives through
      # the D-updates — the difference between fitting BigGAN-128 at 256 images per GPU in 180 GB and not.
      def gen(i, record):
        f = self.inputs[i]
        sy = self._get_one_hot_labels(f["sampled_labels"]) if self.conditional else None
        with tape.record(record):
          return self.generator(f["z"], y=sy, is_training=True)
      d_params = self.store.trainable_under("discriminator")
      g_params = self.store.trainable_under("generator")
      ones = K.fill_(K.empty(1), 1.0)
      for i in range(k):                                # _train_discriminator (:471-485)
        f = dict(self.inputs[i])
        f["generated"] = tape.DT(gen(i, False).t)       # tf.stop_gradient
        self.create_loss(f, f.get("labels"), for_discriminator=True)
        grads = tape.backward([(self.d_loss, ones)], list(d_params.values()), K.add_grad,
                              sinks=self._grad_sinks("discriminator", d_params))
        scale = self._apply_grads("discriminator", self.flat_d, grads, list(d_params.keys()))
        self.d_opt.apply(scale)
        K._call("copy", self.losses.ptr + 4 * i, self.d_loss.ptr, 1)
        self.d_loss = self.g_loss = None
      f = dict(self.inputs[k])                          # _train_generator (:487-510)
      f["generated"] = gen(k, True)
      self.create_loss(f, f.get("labels"), for_discriminator=False)
      grads = tape.backward([(self.g_loss, ones)], list(g_params.values()), K.add_grad,
                            sinks=self._grad_sinks("generator", g_params))
      scale = self._apply_grads("generator", self.flat_g, grads, list(g_params.keys()))
      self.g_opt.apply(scale, self.ema, self._ema_decay, self._ema_start_step)
      K._call("copy", self.losses.ptr + 4 * k, self.g_loss.ptr, 1)
      self.d_loss = self.g_loss = None

  def _substep(self):
    """One step of the NON-unrolled schedule (reference model_fn with unroll_graph False, :534-535, 566-575 — the
    reference's default off TPU): ONE batch, one generator forward, one discriminator update, and a generator update only
    when the discriminator step counter reaches a multiple of disc_iters (`tf.cond(disc_step % disc_iters == 0, ...)`,
    evaluated after the D update).  Uses input slot 0; the device step counters advance exactly as in TF (global_step
    counts G updates, global_step_disc D updates).  Returns True when the G update ran.  Eager only: the branch is taken
    on the host from a mirror of the device counter (one 4-byte read), which is what makes it uncapturable."""
    k = self._disc_iters
    will_g = (int(self.d_opt.step.item()) + 1) % k == 0
    with V.use(self.store):
      f = dict(self.inputs[0])
      sy = self._get_one_hot_labels(f["sampled_labels"]) if self.conditional else None
      with tape.record(will_g):
        gen = self.generator(f["z"], y=sy, is_training=True)          # _split_inputs_and_generate_samples, one sub-step
      d_params = self.store.trainable_under("discriminator")
      g_params = self.store.trainable_under("generator")
      ones = K.fill_(K.empty(1), 1.0)
      f["generated"] = tape.DT(gen.t)                                   # tf.stop_gradient (:476)
      self.create_loss(f, f.get("labels"), for_discriminator=True)
      grads = tape.backward([(self.d_loss, ones)], list(d_params.values()), K.add_grad,
                            sinks=self._grad_sinks("discriminator", d_params))
      scale = self._apply_grads("discriminator", self.flat_d, grads, list(d_params.keys()))
      self.d_opt.apply(scale)
      K._call("copy", self.losses.ptr, self.d_loss.ptr, 1)
      self.d_loss = self.g_loss = None
      if will_g:
        f["generated"] = gen
        self.create_loss(f, f.get("labels"), for_discriminator=False)
        grads = tape.backward([(self.g_loss, ones)], list(g_params.values()), K.add_grad,
                              sinks=self._grad_sinks("generator", g_params))
        scale = self._apply_grads("generator", self.flat_g, grads, list(g_params.keys()))
        self.g_opt.apply(scale, self.ema, self._ema_decay, self._ema_start_step)
        K._call("copy", self.losses.ptr + 4 * k, self.g_loss.ptr, 1)
        self.d_loss = self.g_loss = None
    return will_g

  # ---- public step API -------------------------------------------------------------------------------------
  def run_substep(self):
    """One step of the reference's non-unrolled (CPU / GPU default) schedule on input slot 0, see _substep."""
    K.sync_stream()
    return self._substep()

  def set_inputs(self, images, z, labels=None, sampled_labels=None, alphas=None, non_blocking=True):
    """Host -> device copy of one cycle's inputs (lists of length disc_iters+1 of numpy / pinned torch arrays)."""
    def put(dst, src):
      if src is None:
        return
      t = src if torch.is_tensor(src) else torch.from_numpy(np.ascontiguousarray(src))
      dst.t.copy_(t.view(dst.t.shape) if t.numel() == dst.t.numel() else t, non_blocking=non_blocking)
    for i, f in enumerate(self.inputs):
      put(f["images"], images[i])
      put(f["z"], z[i])
      if self.conditional:
        put(f["labels"], labels[i])
        put(f["sampled_labels"], sampled_labels[i])
      if alphas is not None:
        put(f["alpha"], alphas[i])

  def run_cycle(self):
    """Executes one cycle on the current inputs (graph replay when captured).  Asynchronous."""
    if self._graph is not None:
      self._graph.replay()
    else:
      K.sync_stream()
      self._cycle()

  def capture(self, warmup=3):
    """Capture the cycle into a CUDA graph.  State mutated by the warm-up/capture passes is restored."""
    snap = self.snapshot()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      K.sync_stream()
      for _ in range(warmup):
        self._cycle()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    # the warm-up's activation memory sits cached in the default pool; the graph allocates from its own private pool, so
    # hand the cache back to the driver first (otherwise the peak is paid twice: BigGAN-128 at 256/GPU would not fit)
    torch.cuda.empty_cache()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      K.sync_stream()
      self._cycle()
    K.sync_stream()
    torch.cuda.synchronize()
    self._graph = g
    self.restore(snap)
    return g

  def read_losses(self):
    """(d_losses list, g_loss) of the last cycle — a device->host read (synchronises)."""
    a = self.losses.t.cpu().numpy()
    return [float(x) for x in a[:-1]], float(a[-1])

  @property
  def global_step(self):
    return int(self.g_opt.step.item())

  @property
  def global_step_disc(self):
    return int(self.d_opt.step.item())

  # ---- state I/O (checkpoint key space = reference variable names) ------------------------------------------
  def snapshot(self):
    s = {"vars": {k: v.t.clone() for k, v in self.store.vars.items()},
         "g": (self.g_opt.m.t.clone(), self.g_opt.v.t.clone(), self.g_opt.step.clone()),
         "d": (self.d_opt.m.t.clone(), self.d_opt.v.t.clone(), self.d_opt.step.clone()),
         "ema": None if self.ema is None else self.ema.t.clone(), "losses": self.losses.t.clone()}
    return s

  def restore(self, s):
    for k, v in self.store.vars.items():
      v.t.copy_(s["vars"][k])
    for opt, key in ((self.g_opt, "g"), (self.d_opt, "d")):
      opt.m.t.copy_(s[key][0]); opt.v.t.copy_(s[key][1]); opt.step.copy_(s[key][2])
    if self.ema is not None:
      self.ema.t.copy_(s["ema"])
    self.losses.t.copy_(s["losses"])
    torch.cuda.synchronize()

  # Checkpoints use the reference's variable key space (SURVEY §5): model variables under their TF names, Adam slots as
  # `<var>/Adam`, `<var>/Adam_1`, EMA shadows as `<var>/ExponentialMovingAverage`, plus global_step / global_step_disc.
  def checkpoint_dict(self):
    out = dict(self.store.state_numpy())
    for prefix, flat, opt in (("generator", self.flat_g, self.g_opt), ("discriminator", self.flat_d, self.d_opt)):
      m, v = opt.m.cpu(), opt.v.cpu()
      ema = self.ema.cpu() if (prefix == "generator" and self.ema is not None) else None
      for name, (off, n) in flat["views"].items():
        shape = self.store.vars[name].shape
        out[name + "/Adam"] = m[off:off + n].reshape(shape).copy()
        out[name + "/Adam_1"] = v[off:off + n].reshape(shape).copy()
        if ema is not None:
          out[name + "/ExponentialMovingAverage"] = ema[off:off + n].reshape(shape).copy()
    out["global_step"] = np.array(self.global_step, np.int64)
    out["global_step_disc"] = np.array(self.global_step_disc, np.int64)
    return out

  def save_checkpoint(self, model_dir):
    import os
    os.makedirs(model_dir, exist_ok=True)
    path = os.path.join(model_dir, "model.ckpt-%d.npz" % self.global_step)
    np.savez(path, **{k.replace("/", "|"): v for k, v in self.checkpoint_dict().items()})
    return path

  def load_checkpoint(self, path):
    """Restores model variables, Adam slots, EMA shadows and the step counters from this package's `.npz` or from a
    TensorFlow V2 checkpoint written by the reference (`model.ckpt-<step>`: the prefix, its `.index` or a directory holding
    checkpoints) — the variable names are the same key space (tf_checkpoint.py)."""
    import os
    if path.endswith(".npz"):
      data = {k.replace("|", "/"): v for k, v in np.load(path).items()}
    else:
      from .. import tf_checkpoint
      prefix = path[:-len(".index")] if path.endswith(".index") else path
      if os.path.isdir(prefix):
        prefix = tf_checkpoint.latest_checkpoint(prefix)
        if prefix is None:
          raise ValueError("no model.ckpt-<step>.index under %s" % path)
      data = tf_checkpoint.load_checkpoint(prefix)
      missing = [k for k in self.store.vars if k not in data and not k.endswith("update_accus")]
      if missing:
        raise ValueError("TensorFlow checkpoint %s lacks %d variables of this model, e.g. %s" % (prefix, len(missing), missing[:3]))
      data.setdefault("global_step_disc", np.array(0, np.int64))
    self.store.load_numpy({k: v for k, v in data.items() if k in self.store.vars})
    for prefix, flat, opt in (("generator", self.flat_g, self.g_opt), ("discriminator", self.flat_d, self.d_opt)):
      m, v = opt.m.cpu(), opt.v.cpu()
      ema = self.ema.cpu() if (prefix == "generator" and self.ema is not None) else None
      for name, (off, n) in flat["views"].items():
        if name + "/Adam" in data:
          m[off:off + n] = data[name + "/Adam"].ravel()
          v[off:off + n] = data[name + "/Adam_1"].ravel()
        if ema is not None and name + "/ExponentialMovingAverage" in data:
          ema[off:off + n] = data[name + "/ExponentialMovingAverage"].ravel()
      opt.m.t.copy_(torch.from_numpy(m)); opt.v.t.copy_(torch.from_numpy(v))
      if ema is not None:
        self.ema.t.copy_(torch.from_numpy(ema))
    # TF counts sub-steps differently on CPU/GPU (non-unrolled: one global_step per D or G update); the counters are only
    # used for Adam's bias correction and the EMA start here
    self.g_opt.step.fill_(int(data["global_step"]))
    self.d_opt.step.fill_(int(data["global_step_disc"]))
    torch.cuda.synchronize()

  def state_numpy(self):
    return self.store.state_numpy()

  def load_numpy(self, state):
    self.store.load_numpy(state)
    if self.ema is not None:
      self.ema.t.copy_(self.flat_g["param"].t)


from . import ssgan  # noqa: E402,F401  (registers @SSGAN with gin wherever ModularGAN is importable)
from . import s3gan  # noqa: E402,F401  (registers @S3GAN)
