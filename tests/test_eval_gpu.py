"""Evaluation path parity: TF-style bilinear resize, Inception-v3 features, and the FID / IS / KID numbers of a tiny
generator, engine (CUDA) vs the CPU oracle with the SAME synthetic Inception weights."""
import numpy as np
import pytest
import torch

from oracle import inception as oinc
from oracle import metrics as ometrics
from tests.gpu_util import assert_close, make_pair

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
  from compare_gan_b200 import kernels
  kernels.init(0)
  return kernels


def test_resize_bilinear_matches_tf_semantics(K):
  rng = np.random.RandomState(0)
  for (h, oh) in [(32, 299), (128, 299), (5, 7), (300, 299)]:
    x = rng.rand(2, h, h, 3).astype(np.float32)
    ref = oinc.resize_bilinear_tf(torch.from_numpy(x), oh, oh).numpy()
    got = K.resize_bilinear(K.from_numpy(x), oh, oh).cpu()
    assert_close(got, ref, 1e-5, "resize %d->%d" % (h, oh))
  x = rng.rand(2, 32, 32, 3).astype(np.float32)
  got = K.resize_bilinear(K.from_numpy(x), 299, 299, inception_scale=True).cpu()
  assert_close(got, oinc.preprocess(x).numpy(), 1e-5, "inception preprocessing")


def test_pool2d_tf_semantics(K):
  rng = np.random.RandomState(1)
  x = rng.randn(2, 9, 9, 5).astype(np.float32)
  for mode, k, s, pad in [("max", 3, 2, "VALID"), ("avg", 3, 1, "SAME"), ("max", 3, 1, "SAME")]:
    ref = oinc._pool(torch.from_numpy(x), mode, k, s, pad).numpy()
    got = K.pool2d(K.from_numpy(x), k, s, pad, mode).cpu()
    assert_close(got, ref, 1e-6, "pool %s %s" % (mode, pad))


def test_inception_v3_features(K):
  from compare_gan_b200 import inception
  assert inception.POOL_DIM == 2048 and inception.NUM_CLASSES == 1008
  assert abs(inception.flops_per_image() / 1e9 - 11.4) < 0.6      # SURVEY §2.2 K13: ~11.4 GF / image
  w = inception.synthetic_weights(0)
  net = inception.InceptionV3(w)
  rng = np.random.RandomState(2)
  x = (rng.rand(2, 299, 299, 3).astype(np.float32) * 2 - 1)
  pool, logits = net(K.from_numpy(x))
  rp, rl = oinc.inception_v3(x, w)
  assert pool.shape == (2, 2048) and logits.shape == (2, 1008)
  assert_close(pool.cpu(), rp.numpy(), 2e-4, "pool_3")
  assert_close(logits.cpu(), rl.numpy(), 2e-4, "logits")


def test_eval_fid_is_kid_against_oracle(K):
  from compare_gan_b200 import eval_gan_lib, eval_utils, inception
  from compare_gan_b200.metrics import fid_score, inception_score, kid_score
  eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True)
  tasks = [fid_score.FIDScoreTask(), inception_score.InceptionScoreTask(), kid_score.KIDScoreTask()]
  n = 96
  rng = np.random.RandomState(3)
  real = rng.rand(n, 32, 32, 3).astype(np.float32)
  res = eval_gan_lib.evaluate(eng, tasks, num_averaging_runs=1, num_samples=n, batch_size=32, seed=42, real_images=real)
  assert res["eval_samples_per_sec"] > 0
  for key in ("fid_score", "inception_score", "kid_score"):
    assert key + "_mean" in res and key + "_std" in res and key + "_list" in res      # eval_gan_lib_test.py:78-120
  # oracle: regenerate the same samples (same z stream) with the engine's generator, then features + metrics on the CPU
  from compare_gan_b200 import runner_lib
  rs = np.random.RandomState(42)
  w = eval_utils.get_inception().host_weights
  fake_acts, fake_logits = [], []
  for _ in range(n // 32):
    imgs = eval_gan_lib.generate_batch(eng, 32, rs).cpu()
    p, l = oinc.inception_v3(oinc.preprocess(imgs), w)
    fake_acts.append(p.numpy()); fake_logits.append(l.numpy())
  ra, _ = oinc.inception_v3(oinc.preprocess(real), w)
  fa, fl, ra = np.concatenate(fake_acts), np.concatenate(fake_logits), ra.numpy()
  fid_ref = ometrics.compute_fid_from_activations(ra, fa)
  is_ref = ometrics.inception_score_from_logits(fl)
  kid_ref = ometrics.kid(fa, ra)
  assert abs(res["fid_score_mean"] - fid_ref) <= 5e-3 * abs(fid_ref), (res["fid_score_mean"], fid_ref)     # +-0.5 %
  assert abs(res["inception_score_mean"] - is_ref) <= 5e-3 * abs(is_ref), (res["inception_score_mean"], is_ref)
  assert abs(res["kid_score_mean"] - kid_ref) <= 5e-3 * abs(kid_ref) + 1e-6, (res["kid_score_mean"], kid_ref)


def test_inception_v3_features_tf32(K):
  """math_mode 1: the stride-1 SAME convolutions of Inception (35x35 / 17x17 / 8x8 maps, 1x7 / 7x1 / 5x5 kernels, 48/80-
  channel inputs) run on the tensor cores through border-overhanging 128-pixel boxes and zero-padded K; pool_3 within 2e-3."""
  from compare_gan_b200 import inception
  w = inception.synthetic_weights(0)
  rng = np.random.RandomState(2)
  x = (rng.rand(2, 299, 299, 3).astype(np.float32) * 2 - 1)
  rp, rl = oinc.inception_v3(x, w)
  K.set_math_mode(1)
  try:
    net = inception.InceptionV3(w)
    n0 = K.lib().launch_count()
    pool, logits = net(K.from_numpy(x))
    assert K.lib().launch_count() - n0 > 94
  finally:
    K.set_math_mode(0)
  assert_close(pool.cpu(), rp.numpy(), 2e-3, "pool_3 (tf32)")
  assert_close(logits.cpu(), rl.numpy(), 3e-3, "logits (tf32)")


def test_eval_cuda_graph_equals_eager(K):
  """The CUDA-graph-captured evaluation batch must give exactly the statistics of the eager path."""
  from compare_gan_b200 import eval_gan_lib
  from compare_gan_b200.metrics import fid_score, inception_score
  eng, _ = make_pair("resnet_cifar_arch", (32, 32, 3), 4, d_sn=True)
  tasks = [fid_score.FIDScoreTask(), inception_score.InceptionScoreTask()]
  real = np.random.RandomState(5).rand(64, 32, 32, 3).astype(np.float32)
  kw = dict(num_averaging_runs=1, num_samples=144, batch_size=32, seed=7, real_images=real)
  a = eval_gan_lib.evaluate(eng, tasks, use_graph=True, **kw)
  b = eval_gan_lib.evaluate(eng, tasks, use_graph=False, **kw)
  assert a["fid_score_mean"] == b["fid_score_mean"] and a["inception_score_mean"] == b["inception_score_mean"]


def test_eval_after_train_schedule_and_checkpoint_roundtrip(K, tmp_path):
  """runner_lib.run_with_schedule("eval_after_train") (reference runner_lib_test.py:149-255): trains a few cycles, writes
  model.ckpt-<step>.npz in the reference's variable key space + operative_config-0.gin + TRAIN_DONE, evaluates the
  checkpoint and appends a row to scores.csv; loading the checkpoint restores the state bit for bit."""
  import csv, os
  from compare_gan_b200 import configs, gin_lite as gin, runner_lib
  from compare_gan_b200.gans import modular_gan  # noqa: F401
  gin.clear_config()
  gin.parse_config(configs.RESNET_CIFAR10)
  gin.parse_config("options.batch_size = 8\nModularGAN.g_use_ema = True\nModularGAN.ema_start_step = 0")
  md = str(tmp_path / "run")
  out = runner_lib.run_with_schedule("eval_after_train", model_dir=md, num_cycles=2, use_graph=False,
                                     eval_kwargs=dict(num_samples=64, num_averaging_runs=1))
  gan = out["gan"]
  assert os.path.exists(os.path.join(md, "TRAIN_DONE")) and os.path.exists(os.path.join(md, "operative_config-0.gin"))
  ckpt = os.path.join(md, "model.ckpt-2.npz")
  assert os.path.exists(ckpt)
  keys = set(k.replace("|", "/") for k in np.load(ckpt).keys())
  for k in ("generator/B1/up_conv1/kernel", "generator/B1/up_conv1/kernel/Adam", "generator/B1/up_conv1/kernel/Adam_1",
            "generator/B1/up_conv1/kernel/ExponentialMovingAverage", "discriminator/B1/same_conv1/kernel/u_var",
            "generator/B1/bn1/moving_mean", "global_step", "global_step_disc"):
    assert k in keys, k
  rows = list(csv.DictReader(open(os.path.join(md, "scores.csv"))))
  assert len(rows) == 1 and rows[0]["step"] == "2" and "fid_score_mean" in rows[0] and "inception_score_mean" in rows[0]
  before = gan.checkpoint_dict()
  gan.store.vars["generator/fc_noise/kernel"].t.zero_()
  gan.g_opt.m.t.zero_()
  gan.load_checkpoint(ckpt)
  after = gan.checkpoint_dict()
  for k in before:
    np.testing.assert_array_equal(before[k], after[k], err_msg=k)


def test_train_from_input_pipeline(K, tmp_path):
  """run_with_schedule("train", input_pipeline=True): every cycle takes disc_iters+1 batches from
  dataset.train_input_fn (the reference's fake data set through the native prefetching loader, datasets.py:136-145,
  261-291).  The images resident on the device after the last cycle are exactly the batches the tf.data model of the
  shuffle stream predicts for that cycle."""
  from compare_gan_b200 import configs, datasets, gin_lite as gin, runner_lib
  from compare_gan_b200.gans import modular_gan  # noqa: F401
  from tests.test_input_pipeline import model_stream
  gin.clear_config()
  gin.parse_config(configs.RESNET_CIFAR10)
  gin.parse_config("options.batch_size = 8")
  out = runner_lib.run_with_schedule("train", model_dir=str(tmp_path / "run"), num_cycles=3, use_graph=False,
                                     input_pipeline=True)
  gan = out["gan"]
  assert np.isfinite(out["g_loss"]) and all(np.isfinite(v) for v in out["d_loss"])
  k1 = gan._disc_iters + 1
  ds = datasets.get_dataset()
  fake, _ = ds._make_fake_dataset("train")
  ids = model_stream(len(fake), 10000, 547, 3 * k1 * 8)
  for i in range(k1):
    want = fake[ids[(2 * k1 + i) * 8:(2 * k1 + i + 1) * 8]]
    np.testing.assert_array_equal(gan.inputs[i]["images"].cpu(), want)


@pytest.mark.parametrize("case", ["moving_averages", "accumulators_and_ema"])
def test_inference_mode_generator_and_eval_loop_match_the_oracle(K, case):
  """The evaluation hand-off of the reference (eval_gan_lib.py:65-212, modular_gan.py:266-285) against its oracle
  restatement (oracle/eval.py), from IDENTICAL trained state: the generator in inference mode reads the BN moving
  averages (resnet_cifar10.gin) or the accumulators filled by `_update_bn_accumulators` with the EMA shadows swapped in
  for the weights (biggan_imagenet128.gin); then the whole loop — seed, z / label stream, batches, fake data sets,
  Inception features, FID / IS / KID — within the +-0.5 % north_star states."""
  from compare_gan_b200 import eval_gan_lib, eval_utils
  from compare_gan_b200.metrics import fid_score, inception_score, kid_score
  from oracle import eval as oeval
  from tests.gpu_util import make_inputs
  if case == "moving_averages":
    eng, orc = make_pair("resnet_cifar_arch", (32, 32, 3), 8, d_sn=True, disc_iters=1)
    nc, zd = 0, 128
  else:
    eb = ["resnet_biggan.Generator.blocks_with_attention = 'B2'", "resnet_biggan.Discriminator.blocks_with_attention = 'B1'"]
    eng, orc = make_pair("resnet_biggan_arch", (32, 32, 3), 8, loss="hinge", disc_iters=1, g_bn="conditional_batch_norm",
                         g_sn=True, d_sn=True, sn_singular="auto", conditional=True, num_classes=10, initializer="orthogonal",
                         use_moving_averages=False, g_lr=1e-3, d_lr=5e-4, beta1=0.0, beta2=0.999, z_dim=120, g_use_ema=True,
                         ema_start_step=0, ch=8, extra_bindings=eb, project_y=True)
    nc, zd = 10, 120
  rng = np.random.RandomState(2)
  for _ in range(2):          # the state the evaluation reads must differ from its initial values
    eng.set_inputs(*make_inputs(rng, 1, 8, (32, 32, 3), zd, nc))
    eng.run_cycle()
  eng.read_losses()
  orc._ensure_opts()
  orc.store.load_numpy(eng.state_numpy())
  if eng.ema is not None:
    shadow = eng.ema.cpu()
    assert not np.array_equal(shadow, eng.flat_g["param"].cpu()), "EMA shadows should differ from the weights here"
    for name, (off, n) in eng.flat_g["views"].items():
      orc.ema[name] = torch.from_numpy(shadow[off:off + n].reshape(orc.ema[name].shape).copy())
  # (a) the accumulator pass and one inference batch, same RNG stream on both sides
  with eval_gan_lib.use_ema_weights(eng):
    r = np.random.RandomState(42)
    had = eval_gan_lib._update_bn_accumulators(eng, 8, 48, r)
    imgs = eval_gan_lib.generate_batch(eng, 8, r).cpu()
  with oeval._EmaWeights(orc):
    r = np.random.RandomState(42)
    ohad = oeval.update_bn_accumulators(orc, 8, 48, r)
    oimgs = oeval.sample_batch(orc, 8, r).numpy()
  assert had == ohad == (case != "moving_averages")
  assert_close(imgs, oimgs, 5e-4, "inference-mode generator (%s)" % case)
  if had:
    es = eng.state_numpy()
    for k, v in orc.store.vars.items():
      if "/accu/" in k:
        assert_close(es[k], v.numpy(), 1e-4, k)
    assert float(es["generator/B1/bn1/accu/accu_counter"]) == pytest.approx(6.0)
  # weights are back in place after the EMA swap
  np.testing.assert_array_equal(eng.state_numpy()["generator/fc_noise/kernel"], orc.store.vars["generator/fc_noise/kernel"].detach().numpy())
  # (b) the whole loop
  n = 64
  real = np.random.RandomState(3).rand(n, 32, 32, 3).astype(np.float32)
  tasks = [fid_score.FIDScoreTask(), inception_score.InceptionScoreTask(), kid_score.KIDScoreTask()]
  res = eval_gan_lib.evaluate(eng, tasks, num_averaging_runs=2, num_samples=n, batch_size=16, seed=42, real_images=real,
                              num_accu_examples=48, use_graph=False)
  ref, _ = oeval.evaluate(orc, eval_utils.get_inception().host_weights, real, n, batch_size=16, seed=42,
                          num_averaging_runs=2, num_accu_examples=48)
  for key in ("fid_score", "inception_score", "kid_score"):
    a, b = res[key + "_mean"], ref[key + "_mean"]
    assert abs(a - b) <= 5e-3 * abs(b) + (1e-6 if key == "kid_score" else 0), (key, a, b)
    assert len(res[key + "_list"].split("_")) == 2
