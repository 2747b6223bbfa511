"""Oracle (test infrastructure): losses, penalties, TF-form Adam, EMA and one
ModularGAN training cycle (disc_iters D-updates + 1 G-update, unrolled/TPU
semantics) restated on PyTorch-CPU.
"""
from collections import OrderedDict

import numpy as np
import torch

from . import nets
from . import tf_ops as T


# --------------------------------------------------------------------------- loss_lib

def _check_pair(a, b):
  if tuple(a) != tuple(b):
    raise ValueError("Shape mismatch: %s vs %s." % (tuple(a), tuple(b)))
  if len(a) != 2 or len(b) != 2:
    raise ValueError("Rank: expected 2, got %s and %s" % (len(a), len(b)))


def _relu(x):
  """tf.nn.relu with ReluGrad's gradient, 0 at the kink x = 0 (torch.clamp would pass 1 there)."""
  return torch.where(x > 0, x, torch.zeros_like(x))


def get_losses(fn, d_real, d_fake, d_real_logits, d_fake_logits):
  """gans/loss_lib.py:53-154 -> (d_loss, d_loss_real, d_loss_fake, g_loss)."""
  _check_pair(d_real_logits.shape, d_fake_logits.shape)
  if fn == "non_saturating":      # :53-78
    lr = T.sigmoid_ce(d_real_logits, True).mean()
    lf = T.sigmoid_ce(d_fake_logits, False).mean()
    return lr + lf, lr, lf, T.sigmoid_ce(d_fake_logits, True).mean()
  if fn == "wasserstein":         # :81-101
    lr = -d_real_logits.mean()
    lf = d_fake_logits.mean()
    return lr + lf, lr, lf, -lf
  if fn == "least_squares":       # :104-124
    lr = ((d_real - 1.0) ** 2).mean()
    lf = (d_fake ** 2).mean()
    return 0.5 * (lr + lf), lr, lf, 0.5 * ((d_fake - 1.0) ** 2).mean()
  if fn == "hinge":               # :127-148
    lr = _relu(1.0 - d_real_logits).mean()
    lf = _relu(1.0 + d_fake_logits).mean()
    return lr + lf, lr, lf, -d_fake_logits.mean()
  raise ValueError(fn)


# --------------------------------------------------------------------------- penalty_lib

def wgangp_penalty(store, cfg, x, x_fake, y, is_training, alpha):
  """gans/penalty_lib.py:59-82; ``alpha`` [B,1,1,1] is fed (SURVEY §5 RNG)."""
  xi = (x + alpha * (x_fake - x)).detach().requires_grad_(True)
  logits = nets.discriminator(store, cfg, xi, y, is_training)[1]
  g = torch.autograd.grad(logits.sum(), xi, create_graph=True)[0]
  slopes = torch.sqrt(0.0001 + (g * g).sum(dim=(1, 2, 3)))
  return ((slopes - 1.0) ** 2).mean()


def get_penalty_loss(fn, store, cfg, x, x_fake, y, is_training, alpha=None):
  """gans/penalty_lib.py:105-108."""
  if fn == "no_penalty":
    return torch.zeros(())
  if fn == "wgangp_penalty":
    return wgangp_penalty(store, cfg, x, x_fake, y, is_training, alpha)
  raise ValueError(fn)


# --------------------------------------------------------------------------- optimizer

class TFAdam(object):
  """tf.train.AdamOptimizer: lr_t = lr*sqrt(1-b2^t)/(1-b1^t);
  theta -= lr_t*m/(sqrt(v)+eps), eps=1e-8 outside the corrected sqrt."""

  def __init__(self, params, lr, beta1, beta2, eps=1e-8):
    self.params = params            # OrderedDict name -> tensor
    self.lr, self.b1, self.b2, self.eps = lr, beta1, beta2, eps
    self.m = OrderedDict((k, torch.zeros_like(v)) for k, v in params.items())
    self.v = OrderedDict((k, torch.zeros_like(v)) for k, v in params.items())
    self.t = 0

  def step(self, grads):
    self.t += 1
    lr_t = self.lr * np.sqrt(1.0 - self.b2 ** self.t) / (1.0 - self.b1 ** self.t)
    lr_t = np.float32(lr_t)
    with torch.no_grad():
      for k, p in self.params.items():
        g = grads[k]
        self.m[k].mul_(self.b1).add_(g, alpha=1.0 - self.b1)
        self.v[k].mul_(self.b2).addcmul_(g, g, value=1.0 - self.b2)
        p.sub_(lr_t * self.m[k] / (self.v[k].sqrt() + self.eps))


# --------------------------------------------------------------------------- ModularGAN cycle

class GanOracle(object):
  """gans/modular_gan.py restated (model_fn :512-604, create_loss :618-670)."""

  def __init__(self, cfg, loss="non_saturating", penalty="no_penalty", lamba=1.0, disc_iters=1,
               g_lr=2e-4, d_lr=None, beta1=0.5, beta2=0.999, conditional=False,
               g_use_ema=False, ema_decay=0.9999, ema_start_step=40000, z_dim=128, seed=0,
               dtype=torch.float32):
    self.cfg, self.loss, self.penalty = cfg, loss, penalty
    self.lamba, self.disc_iters = lamba, disc_iters
    self.g_lr, self.d_lr = g_lr, g_lr if d_lr is None else d_lr
    self.beta1, self.beta2 = beta1, beta2
    self.conditional = conditional
    self.g_use_ema, self.ema_decay, self.ema_start_step = g_use_ema, ema_decay, ema_start_step
    self.z_dim = z_dim
    self.dtype = dtype
    self.store = nets.VarStore(seed, dtype)
    self.global_step = 0        # counts G steps  (modular_gan_test.py:175-177)
    self.global_step_disc = 0   # counts D steps
    self.d_opt = self.g_opt = None
    self.ema = None

  def one_hot(self, labels):
    return torch.nn.functional.one_hot(torch.as_tensor(labels).long(),
                                       self.cfg.num_classes).to(self.dtype)

  def build(self, batch):
    """Create all variables by one G and one D call (like TF graph construction)."""
    h, w, c = self.cfg.image_shape
    z = torch.zeros(batch, self.z_dim, dtype=self.dtype)
    y = self.one_hot(np.zeros(batch, np.int64)) if self.conditional else None
    with torch.no_grad():
      x = nets.generator(self.store, self.cfg, z, y, True)
      nets.discriminator(self.store, self.cfg, torch.cat([x, x]),
                         None if y is None else torch.cat([y, y]), True)
      # graph construction runs no ops in TF: undo the moving-average / u_var side effects
      for k, v in self.store.vars.items():
        if k.endswith("moving_mean"):
          v.zero_()
        elif k.endswith("moving_variance"):
          v.fill_(1.0)
    return self

  def _ensure_opts(self):
    if self.d_opt is None:
      self.d_opt = TFAdam(self.store.trainable_under("discriminator"), self.d_lr, self.beta1, self.beta2)
      self.g_opt = TFAdam(self.store.trainable_under("generator"), self.g_lr, self.beta1, self.beta2)
      if self.g_use_ema:
        self.ema = OrderedDict((k, v.detach().clone())
                               for k, v in self.store.trainable_under("generator").items())

  def create_loss(self, images, generated, y, sampled_y, alpha=None, for_d=True):
    """modular_gan.py:618-670: D on concat([real, fake]) as ONE batch of 2B."""
    all_images = torch.cat([images, generated], 0)
    all_y = torch.cat([y, sampled_y], 0) if self.conditional else None
    d_all, d_all_logits, _ = nets.discriminator(self.store, self.cfg, all_images, all_y, True)
    b = images.shape[0]
    d_loss, _, _, g_loss = get_losses(self.loss, d_all[:b], d_all[b:], d_all_logits[:b], d_all_logits[b:])
    if not for_d:   # g_loss does not depend on the penalty sub-graph, TF never runs it
      return None, g_loss
    pen = get_penalty_loss(self.penalty, self.store, self.cfg, images, generated, y, True, alpha)
    return d_loss + self.lamba * pen, g_loss

  def cycle(self, images, z, labels=None, sampled_labels=None, alphas=None):
    """One unrolled cycle.  images/z/...: lists of length disc_iters+1 (one per sub-step)."""
    self._ensure_opts()
    k = self.disc_iters
    ys = [self.one_hot(l) for l in labels] if self.conditional else [None] * (k + 1)
    sys_ = [self.one_hot(l) for l in sampled_labels] if self.conditional else [None] * (k + 1)
    # _split_inputs_and_generate_samples :428-469.  The reference builds all k+1 G forwards up front; G's weights do not
    # change before the last sub-step, so evaluating sample i right before it is consumed gives identical values (the
    # G calls still happen in the order 0..k, which is what the BN moving averages see).
    def gen_sample(i, grad):
      with torch.set_grad_enabled(grad):     # only the G-step sample needs a backward graph
        return nets.generator(self.store, self.cfg, torch.as_tensor(z[i]).to(self.dtype), sys_[i], True)
    d_losses = []
    for i in range(k):                                  # _train_discriminator :471-485
      gen = gen_sample(i, False).detach()
      d_loss, _ = self.create_loss(torch.as_tensor(images[i]).to(self.dtype), gen, ys[i], sys_[i],
                                   None if alphas is None else torch.as_tensor(alphas[i]).to(self.dtype))
      params = getattr(self, "_d_params", None) or self.store.trainable_under("discriminator")
      grads = torch.autograd.grad(d_loss, list(params.values()), allow_unused=True)
      self.last_d_grads = OrderedDict((n, torch.zeros_like(p) if g is None else g.detach().clone())
                                      for (n, p), g in zip(params.items(), grads))
      self.d_opt.step({n: (g if g is not None else torch.zeros_like(p))
                       for (n, p), g in zip(params.items(), grads)})
      self.global_step_disc += 1
      d_losses.append(float(d_loss.detach()))
    # _train_generator :487-510 — new D forward with updated D, G grads only.
    _, g_loss = self.create_loss(torch.as_tensor(images[k]).to(self.dtype), gen_sample(k, True), ys[k], sys_[k],
                                 None, for_d=False)
    params = self.store.trainable_under("generator")
    grads = torch.autograd.grad(g_loss, list(params.values()), allow_unused=True)
    self.last_g_grads = OrderedDict((n, torch.zeros_like(p) if g is None else g.detach().clone())
                                    for (n, p), g in zip(params.items(), grads))
    self.g_opt.step({n: (g if g is not None else torch.zeros_like(p))
                     for (n, p), g in zip(params.items(), grads)})
    if self.g_use_ema:                                  # :498-508
      decay = self.ema_decay * float(self.global_step >= self.ema_start_step)
      with torch.no_grad():
        for n, p in params.items():
          self.ema[n].sub_((self.ema[n] - p) * (1.0 - decay))
    self.global_step += 1
    return d_losses, float(g_loss.detach())


  def substep(self, images, z, labels=None, sampled_labels=None, alpha=None):
    """One step of the NON-unrolled schedule (modular_gan.py:534-535 num_sub_steps = 1, :566-575): one batch, one G forward
    (its samples feed the D update detached and, when it runs, the G update with gradients), one D update, and the G
    update iff global_step_disc % disc_iters == 0 after the D update.  Returns (d_loss, g_loss or None)."""
    self._ensure_opts()
    y = self.one_hot(labels) if self.conditional else None
    sy = self.one_hot(sampled_labels) if self.conditional else None
    will_g = (self.global_step_disc + 1) % self.disc_iters == 0
    with torch.set_grad_enabled(will_g):
      gen = nets.generator(self.store, self.cfg, torch.as_tensor(z).to(self.dtype), sy, True)
    img = torch.as_tensor(images).to(self.dtype)
    d_loss, _ = self.create_loss(img, gen.detach(), y, sy, None if alpha is None else torch.as_tensor(alpha).to(self.dtype))
    params = self.store.trainable_under("discriminator")
    grads = torch.autograd.grad(d_loss, list(params.values()), allow_unused=True)
    self.d_opt.step({n: (g if g is not None else torch.zeros_like(p)) for (n, p), g in zip(params.items(), grads)})
    self.global_step_disc += 1
    if not will_g:
      return float(d_loss.detach()), None
    _, g_loss = self.create_loss(img, gen, y, sy, None, for_d=False)
    params = self.store.trainable_under("generator")
    grads = torch.autograd.grad(g_loss, list(params.values()), allow_unused=True)
    self.g_opt.step({n: (g if g is not None else torch.zeros_like(p)) for (n, p), g in zip(params.items(), grads)})
    if self.g_use_ema:
      decay = self.ema_decay * float(self.global_step >= self.ema_start_step)
      with torch.no_grad():
        for n, p in params.items():
          self.ema[n].sub_((self.ema[n] - p) * (1.0 - decay))
    self.global_step += 1
    return float(d_loss.detach()), float(g_loss.detach())


# --------------------------------------------------------------------------- SSGAN (gans/ssgan.py)

def rotate_images(images, rot90_scalars=(0, 1, 2, 3)):
  """gans/utils.py:38-49 on NHWC tensors: transpose_image swaps H and W, flip_up_down reverses H, flip_left_right W."""
  tr = lambda x: x.permute(0, 2, 1, 3)
  ud = lambda x: torch.flip(x, dims=[1])
  lr = lambda x: torch.flip(x, dims=[2])
  rotated = [images, ud(tr(images)), lr(ud(images)), tr(ud(images))]
  return torch.cat([rotated[i] for i in rot90_scalars], 0)


class SsganOracle(GanOracle):
  """gans/ssgan.py:40-226 restated: rotation head on the discriminator features, rotation losses for D (real) and G (fake)."""

  def __init__(self, cfg, rotated_batch_size, self_supervision="rotation_gan", weight_rotation_loss_d=1.0,
               weight_rotation_loss_g=0.2, **kw):
    super(SsganOracle, self).__init__(cfg, **kw)
    self.rotated_batch_size, self.self_supervision = rotated_batch_size, self_supervision
    self.w_d, self.w_g = weight_rotation_loss_d, weight_rotation_loss_g

  def _head(self, x, y):
    d, logits, final = nets.discriminator(self.store, self.cfg, x, y, True)
    with self.store.scope("discriminator_rotation"):
      rot = nets.linear(self.store, self.cfg, final.reshape(x.shape[0], -1), 4, "score_classify", use_sn=self.cfg.d_sn)
    return d, logits, rot

  def build(self, batch):
    super(SsganOracle, self).build(batch)
    h, w, c = self.cfg.image_shape
    with torch.no_grad():
      self._head(torch.zeros(2 * batch, h, w, c, dtype=self.dtype), None if not self.conditional else self.one_hot(np.zeros(2 * batch, np.int64)))
    return self

  def _ensure_opts(self):
    if self.d_opt is None:
      d_params = OrderedDict((k, v) for k, v in self.store.trainable.items() if k.split("/")[0].startswith("discriminator"))
      self.d_opt = TFAdam(d_params, self.d_lr, self.beta1, self.beta2)
      self.g_opt = TFAdam(self.store.trainable_under("generator"), self.g_lr, self.beta1, self.beta2)
      self._d_params = d_params

  def create_loss(self, images, generated, y, sampled_y, alpha=None, for_d=True):
    bs = images.shape[0]
    n = self.rotated_batch_size // 4
    rotation = "rotation" in (self.self_supervision or "")
    all_y = None
    if rotation:
      ir = rotate_images(images[bs - n:], (1, 2, 3))
      gr = rotate_images(generated[bs - n:], (1, 2, 3))
      all_images = torch.cat([images, ir, generated, gr], 0)
      if self.conditional:
        yr = y[bs - n:].repeat(3, 1)
        all_y = torch.cat([y, yr, sampled_y, yr], 0)
    else:
      all_images = torch.cat([images, generated], 0)
      if self.conditional:
        all_y = torch.cat([y, sampled_y], 0)
    d_all, d_logits, c_logits = self._head(all_images, all_y)
    half = d_all.shape[0] // 2
    d_loss, _, _, g_loss = get_losses(self.loss, d_all[:bs], d_all[half:half + bs], d_logits[:bs], d_logits[half:half + bs])
    if for_d:
      d_loss = d_loss + self.lamba * get_penalty_loss(self.penalty, self.store, self.cfg, images, generated, y, True, alpha)
    if rotation:
      rb = self.rotated_batch_size
      labels = torch.arange(4).repeat_interleave(n)
      onehot = torch.nn.functional.one_hot(labels, 4).to(self.dtype)
      c_real = -(onehot * torch.log(torch.softmax(c_logits[half - rb:half], -1) + 1e-10)).sum(1).mean()
      c_fake = -(onehot * torch.log(torch.softmax(c_logits[2 * half - rb:], -1) + 1e-10)).sum(1).mean()
      if self.self_supervision == "rotation_only":
        d_loss, g_loss = d_loss * 0.0, g_loss * 0.0
      d_loss = d_loss + c_real * self.w_d
      g_loss = g_loss + c_fake * self.w_g
    return (d_loss if for_d else None), g_loss


# --------------------------------------------------------------------------- S3GAN (gans/s3gan.py)

class S3ganOracle(SsganOracle):
  """gans/s3gan.py:39-321 restated: rotation head (103-134), projection discriminator on real-or-predicted labels (136-158,
  160-173), predictor trained with weighted cross entropy on the labelled real examples (305-318).  No penalty term."""

  def __init__(self, cfg, rotated_batch_fraction=None, self_supervision="rotation", weight_rotation_loss_d=1.0,
               weight_rotation_loss_g=0.2, project_y=False, use_predictor=False, use_soft_pred=False, weight_class_loss=1.0,
               **kw):
    GanOracle.__init__(self, cfg, **kw)
    if use_predictor and not project_y:
      raise ValueError("Using predictor requires projection.")
    self.fraction, self.self_supervision = rotated_batch_fraction, self_supervision
    self.w_d, self.w_g, self.w_class = weight_rotation_loss_d, weight_rotation_loss_g, weight_class_loss
    self.project_y, self.use_predictor, self.use_soft_pred = project_y, use_predictor, use_soft_pred

  def one_hot(self, labels):
    """tf.one_hot: a label of -1 ("no label") gives a row of zeros."""
    lab = torch.as_tensor(labels).long()
    out = torch.zeros(lab.shape[0], self.cfg.num_classes, dtype=self.dtype)
    ok = lab >= 0
    out[ok, lab[ok]] = 1.0
    return out

  def _head(self, x, y):
    d, logits, rep = nets.discriminator(self.store, self.cfg, x, y, True)
    assert rep.dim() == 2
    avail = (y.sum(1, keepdim=True) > 0.5).to(self.dtype) if y is not None else None
    rot = None
    if "rotation" in self.self_supervision:
      with self.store.scope("discriminator_rotation"):
        rot = nets.linear(self.store, self.cfg, rep, 4, "score_classify", use_sn=self.cfg.d_sn)
    if not self.project_y:
      return d, logits, rot, None, avail
    aux = None
    if self.use_predictor:
      with self.store.scope("discriminator_predictor"):
        aux = nets.linear(self.store, self.cfg, rep, y.shape[1], "predictor_linear", use_sn=self.cfg.d_sn, use_bias=True)
      if self.use_soft_pred:
        y_pred = torch.softmax(aux, -1)
      else:
        y_pred = torch.nn.functional.one_hot(aux.argmax(1), aux.shape[1]).to(self.dtype)
      y = ((1.0 - avail) * y_pred + avail * y).detach()
    with self.store.scope("discriminator_projection"):
      k = self.store.get("kernel", (y.shape[1], rep.shape[1]), ("glorot_normal",))
      if self.cfg.d_sn:
        k = nets.spectral_norm(self.store, self.cfg, k)
      emb = y @ k
    logits = logits + (emb * rep).sum(1, keepdim=True)
    return torch.sigmoid(logits), logits, rot, aux, avail

  def build(self, batch):
    GanOracle.build(self, batch)
    h, w, c = self.cfg.image_shape
    with torch.no_grad():
      self._head(torch.zeros(2 * batch, h, w, c, dtype=self.dtype),
                 None if not self.conditional else self.one_hot(np.zeros(2 * batch, np.int64)))
      for k, v in self.store.vars.items():          # graph construction runs no ops (moving averages / u_var untouched)
        if k.endswith("moving_mean"):
          v.zero_()
        elif k.endswith("moving_variance"):
          v.fill_(1.0)
    return self

  def create_loss(self, images, generated, y, sampled_y, alpha=None, for_d=True):
    bs = images.shape[0]
    rotation = self.self_supervision == "rotation"
    n = 0
    if rotation:
      assert bs % self.fraction == 0
      n = (bs // self.fraction) // 4
      assert n > 0
      all_images = torch.cat([images, rotate_images(images[bs - n:], (1, 2, 3)), generated,
                              rotate_images(generated[bs - n:], (1, 2, 3))], 0)
      all_y = torch.cat([y, y[bs - n:].repeat(3, 1), sampled_y, sampled_y[bs - n:].repeat(3, 1)], 0) if self.conditional else None
    else:
      all_images = torch.cat([images, generated], 0)
      all_y = torch.cat([y, sampled_y], 0) if self.conditional else None
    d_all, d_logits, rot, aux, avail = self._head(all_images, all_y)
    half = d_all.shape[0] // 2
    assert d_all.shape[0] == 2 * bs + 6 * n
    d_loss, _, _, g_loss = get_losses(self.loss, d_all[:bs], d_all[half:half + bs], d_logits[:bs], d_logits[half:half + bs])
    if rotation:
      rb = 4 * n
      onehot = torch.nn.functional.one_hot(torch.arange(4).repeat_interleave(n), 4).to(self.dtype)
      real_loss = -(onehot * torch.log(torch.softmax(rot[half - rb:half], -1) + 1e-10)).sum(1).mean()
      fake_loss = -(onehot * torch.log(torch.softmax(rot[2 * half - rb:], -1) + 1e-10)).sum(1).mean()
      d_loss = d_loss + real_loss * self.w_d
      g_loss = g_loss + fake_loss * self.w_g
    if self.use_predictor:
      w = avail[:bs, 0]
      ce = -(y * torch.log_softmax(aux[:bs], -1)).sum(1)
      present = (w != 0).sum()
      class_loss = (w * ce).sum() / present if int(present) > 0 else (w * ce).sum() * 0.0     # SUM_BY_NONZERO_WEIGHTS
      d_loss = d_loss + self.w_class * class_loss
    return (d_loss if for_d else None), g_loss
