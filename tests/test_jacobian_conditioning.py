"""Generator conditioning (reference metrics/jacobian_conditioning.py): the reference's cases, forward-mode tangents of
the generators against float64 Jacobians of the oracle networks (oracle/nets.py), the trace-based check that every op a
generator reaches has a tangent rule, the device entries of csrc/jacobian.cu against float64 formulas, and the metric
inside `evaluate`."""
import numpy as np
import pytest
import torch

from tests.abi_emulator import EmulatedLib, emulated_library


def _jc():
  from compare_gan_b200.metrics import jacobian_conditioning
  return jacobian_conditioning


# ---- the device entries of csrc/jacobian.cu, emulated on the CPU from their header contracts (tests/abi_emulator.py) ----

_EMULATED = {name: getattr(EmulatedLib, name) for name in (
    "cgan_act_jvp", "cgan_bn_apply_jvp", "cgan_maxpool2_jvp", "cgan_softmax_jvp", "cgan_metric_tensor_f64")}


@pytest.fixture
def emulated(monkeypatch):
  for name, fn in _EMULATED.items():
    monkeypatch.setattr(EmulatedLib, name, fn, raising=False)
  from compare_gan_b200 import kernels as K
  with emulated_library():
    yield K


@pytest.fixture(scope="module")
def gpu():
  from compare_gan_b200 import kernels as K
  K.init(0)
  return K


# ---- 1. the reference's cases (jacobian_conditioning_test.py) ----

def check_linear_case(K):
  w = np.array([[2., -1.], [1.5, 1.]], np.float32)
  x = np.random.RandomState(0).standard_normal((32, 2)).astype(np.float32)
  wd = K.from_numpy(w)
  j = _jc().compute_jacobian(lambda xs: K.matmul(xs, wd), x).cpu().numpy()
  assert j.shape == (32, 2, 2) and j.dtype == np.float32
  assert np.array_equal(j, np.tile(w.T[None], (32, 1, 1)))          # f = W^T x in vector notation


def test_linear_case(emulated):
  check_linear_case(emulated)


def test_analyze_jacobian_reference_case(monkeypatch):
  jc = _jc()
  monkeypatch.setattr(jc, "_analyze_metric_tensor", lambda m: m)
  res = jc.analyze_jacobian(np.array([[[1, 2], [3, 4]], [[2, 4], [6, 8]]]))
  assert np.array_equal(res["metric_tensor"], [[[10, 14], [14, 20]], [[40, 56], [56, 80]]])
  assert np.array_equal(res["mean_metric_tensor"], [[[25, 35], [35, 50]]])


def test_analyze_metric_tensor_shapes():
  jac = np.random.RandomState(1).normal(0, 1, (32, 2, 10))
  res = _jc()._analyze_metric_tensor(np.matmul(np.transpose(jac, [0, 2, 1]), jac))
  assert res["eigenvalues"].shape == (32, 10)
  assert res["logdet"].shape == (32,) and res["log_condition_number"].shape == (32,)
  m = np.matmul(np.transpose(jac, [0, 2, 1]), jac)
  assert np.array_equal(_jc().analyze_metric_tensors(m)["metric_tensor"]["logdet"], res["logdet"])


# ---- 2. an MLP three ways: forward mode, reverse mode (one backward per output row, the reference's SlowJacobian) and
#         central differences ----

def _mlp(K, rs):
  shapes = ((2, 20), (20, 20), (20, 10))
  ws = [K.from_numpy((rs.standard_normal(s) / np.sqrt(s[0])).astype(np.float32)) for s in shapes]
  bs = [K.from_numpy((rs.standard_normal(s[1]) * 0.1).astype(np.float32)) for s in shapes]

  def f(x):
    h = K.relu(K.bias_add(K.matmul(x, ws[0]), bs[0]))
    h = K.relu(K.bias_add(K.matmul(h, ws[1]), bs[1]))
    return K.bias_add(K.matmul(h, ws[2]), bs[2])
  return f


def check_mlp_three_ways(K):
  from compare_gan_b200 import tape
  rs = np.random.RandomState(2)
  f = _mlp(K, rs)
  x = rs.standard_normal((32, 2)).astype(np.float32)
  fast = _jc().compute_jacobian(f, x).cpu().numpy()
  slow = np.zeros_like(fast)
  for i in range(10):
    xd = K.from_numpy(x, req=True)
    out = f(xd)
    seed = np.zeros((32, 10), np.float32)
    seed[:, i] = 1
    g, = tape.backward([(out, K.from_numpy(seed))], [xd], K.add_grad)
    slow[:, i, :] = g.cpu()
  np.testing.assert_allclose(fast, slow, rtol=1e-6, atol=1e-6)
  eps = 1e-2                               # piecewise-linear f: exact up to fp32 rounding away from the kinks
  for _ in range(10):
    b, xi, fi = rs.randint(32), rs.randint(2), rs.randint(10)
    xp, xm = x.copy(), x.copy()
    xp[b, xi] += eps
    xm[b, xi] -= eps
    with tape.no_record():
      fp, fm = f(K.from_numpy(xp)).cpu()[b, fi], f(K.from_numpy(xm)).cpu()[b, fi]
    assert abs(fast[b, fi, xi] - (fp - fm) / (2 * eps)) <= 1e-3 * (1 + abs(fast[b, fi, xi])), (b, xi, fi)


def test_mlp_three_ways(emulated):
  check_mlp_three_ways(emulated)


# ---- 3. an op without a tangent rule raises ----

def test_op_without_rule_raises(emulated):
  K = emulated
  from compare_gan_b200 import tape
  x = K.from_numpy(np.ones((2, 4, 4, 3), np.float32))
  x.tan = K.from_numpy(np.ones((6, 4, 4, 3), np.float32))
  with tape.no_record(), K.forward_mode(2, 3):
    with pytest.raises(NotImplementedError, match="globalpool"):
      K.globalpool(x, mean=True)
    with pytest.raises(NotImplementedError, match="concat_rows"):
      K.concat_rows(x, x)
    with pytest.raises(NotImplementedError, match="bn_train"):
      K.bn_train(x, None, None, 1e-5)
    with pytest.raises(NotImplementedError, match="conv2d"):     # a z-dependent weight is not a rule
      K.conv2d(K.from_numpy(np.ones((2, 4, 4, 4), np.float32)), x)
    with pytest.raises(NotImplementedError, match="resize_bilinear"):
      K.resize_bilinear(x, 8, 8)
  with pytest.raises(RuntimeError, match="forward_mode"):
    K.relu(x)


# ---- 4. every op each generator reaches in inference mode has a tangent rule (traced on the CPU) ----

# kernel-layer functions with a tangent rule (kernels.py), and those whose operands are constants of the pass
TANGENT_RULES = {"reshape", "add", "concat_cols", "slice_cols", "conv2d", "deconv2d", "matmul", "bias_add", "relu",
                 "sigmoid", "tanh01", "lrelu", "avgpool2", "unpool", "maxpool2", "scale_by_param", "bn_infer", "bmm",
                 "softmax", "attention"}       # attention: composed of bmm / softmax / bmm in math_mode 0
CONSTANTS = {"spectral_normalize", "one_hot"}


def _inference_ops(case):
  from tests import arch_trace
  from compare_gan_b200 import datasets
  from compare_gan_b200 import gin_lite as gin
  from compare_gan_b200 import variables as V
  from compare_gan_b200.gans import modular_gan
  kw = arch_trace.CASES[case]
  gin.clear_config()
  gin.parse_config(kw["gin_text"])
  shape, nc = kw["image_shape"], kw.get("num_classes", 0)
  ds = datasets.ImageDatasetV2("synthetic", shape[0], shape[2], nc or None, 100)
  params = {"architecture": kw["architecture"], "z_dim": kw.get("z_dim", 128), "lambda": 1, "disc_iters": 1, "seed": 0}
  try:
    with arch_trace.traced_kernels() as tracer:
      gan = modular_gan.ModularGAN(dataset=ds, parameters=params, model_dir="/tmp/arch_trace",
                                   conditional=kw.get("conditional", False))
      z = arch_trace.FakeDT((2, params["z_dim"]))
      y = arch_trace.FakeDT((2, nc)) if kw.get("conditional") else None
      with V.use(V.VariableStore(seed=0)):
        gan.generator(z, y=y, is_training=False)
  finally:
    gin.clear_config()
  return set(op[0] for op in tracer.ops if op[0] != "get_variable")


def test_generator_ops_have_tangent_rules():
  from tests import arch_trace
  archs = set()
  for case, kw in arch_trace.CASES.items():
    ops = _inference_ops(case)
    missing = ops - TANGENT_RULES - CONSTANTS
    assert not missing, (case, sorted(missing))
    archs.add(kw["architecture"])
  assert archs == {"resnet_cifar_arch", "resnet5_arch", "sndcgan_arch", "dcgan_arch", "resnet_biggan_arch",
                   "resnet_biggan_deep_arch"}


# ---- 5. generators against float64 Jacobians of the oracle networks ----

def oracle_jacobian(orc, z, labels):
  """[B, D, k] float64 (or the oracle's dtype): one torch forward-mode product per z column, the oracle's
  non-trainable state restored before every call (its spectral-norm u advances on each)."""
  from oracle import nets as onets
  state = orc.store.state_numpy()
  zt = torch.from_numpy(z).to(orc.dtype)
  y = orc.one_hot(torch.from_numpy(labels).long()) if labels is not None else None
  cols = []
  for j in range(z.shape[1]):
    orc.store.load_numpy(state)
    v = torch.zeros_like(zt)
    v[:, j] = 1

    def f(zz):
      return onets.generator(orc.store, orc.cfg, zz, y, False).reshape(zz.shape[0], -1)
    cols.append(torch.autograd.functional.jvp(f, zt, v)[1].detach())
  orc.store.load_numpy(state)
  return torch.stack(cols, 2).double().numpy()


def _rel(a, b):
  return float(np.linalg.norm(a - b) / np.linalg.norm(b))


# (architecture, image shape, make_pair keywords, z_dim)
GENERATORS = {
    "resnet_cifar": ("resnet_cifar_arch", (32, 32, 3), {}, 8),
    "sndcgan": ("sndcgan_arch", (32, 32, 3), {}, 8),
    "biggan_conditional": ("resnet_biggan_arch", (32, 32, 3),
                           dict(g_bn="conditional_batch_norm", g_sn=True, conditional=True, num_classes=10, ch=8,
                                extra_bindings=("resnet_biggan.Generator.blocks_with_attention = 'B2'",)), 8),
    "resnet5": ("resnet5_arch", (64, 64, 3), {}, 8),
    "dcgan": ("dcgan_arch", (64, 64, 3), {}, 8),
    "biggan_deep": ("resnet_biggan_deep_arch", (64, 64, 3),
                    dict(g_bn="conditional_batch_norm", g_sn=True, conditional=True, num_classes=10, ch=4), 16),
}


def check_generator(K, name, batch=2):
  """J of the tangent pass against the float64 oracle.  Bound: 10x the error of the oracle's own fp32 twin (what fp32
  evaluation of the same network loses) plus 1e-6; log cond(J^T J) within 1e-3."""
  from tests.gpu_util import make_pair
  arch, shape, kw, zd = GENERATORS[name]
  eng, orc32, orc64 = make_pair(arch, shape, batch, z_dim=zd, with64=True, **kw)
  rs = np.random.RandomState(3)
  z, labels = _jc()._draw_latents(eng, batch, rs)
  with _jc()._GeneratorPass(eng) as run:
    imgs, t = run(z, labels)
  got = t.transpose(1, 2).cpu().numpy().astype(np.float64)
  want = oracle_jacobian(orc64, z, labels)
  twin = oracle_jacobian(orc32, z, labels)
  err, err32 = _rel(got, want), _rel(twin, want)
  assert err <= 10 * err32 + 1e-6, (name, err, err32)
  lc = _jc().analyze_jacobian(got)["metric_tensor"]["log_condition_number"]
  lc64 = _jc().analyze_jacobian(want)["metric_tensor"]["log_condition_number"]
  assert np.all(np.abs(lc - lc64) <= 1e-3), (name, lc, lc64)
  return eng, z, labels, imgs


@pytest.mark.parametrize("name", ["resnet_cifar", "sndcgan", "biggan_conditional"])
def test_generator_tangents_match_the_float64_oracle_on_the_emulator(emulated, name):
  check_generator(emulated, name)


# ---- 6. on the H100: the device entries ----

def _dev(a):
  return torch.from_numpy(np.ascontiguousarray(a)).cuda()


GRAM_CASES = ([(3, k, d) for k in (1, 7, 120, 128, 140) for d in (1, 3, 3072, 49152)] +
              [(1, 128, 49152), (1, 7, 3), (64, 128, 3072), (64, 120, 3072), (64, 140, 49152)])


@pytest.mark.gpu
@pytest.mark.parametrize("b,k,d", GRAM_CASES)
def test_metric_tensor_matches_a_float64_gram(gpu, b, k, d):
  rs = np.random.RandomState(b * 7 + k + d)
  t = rs.standard_normal((b, k, d)).astype(np.float32)
  t[:, k // 2] *= 1e-3                           # rows of very different scale
  td = _dev(t)
  m = gpu.metric_tensor_f64(td)
  got = m.cpu().numpy()
  t64 = t.astype(np.float64)
  want = np.matmul(t64, t64.transpose(0, 2, 1))
  diag = np.sqrt(np.einsum("bii->bi", want))
  scale = diag[:, :, None] * diag[:, None, :]
  assert np.all(np.abs(got - want) <= 1e-13 * scale), np.max(np.abs(got - want) / scale)
  assert np.array_equal(got, got.transpose(0, 2, 1))                       # exactly symmetric
  assert torch.equal(m, gpu.metric_tensor_f64(td))                          # bit-identical rerun
  if b > 1:
    assert torch.equal(gpu.metric_tensor_f64(td[1:2].contiguous())[0], m[1])   # a sample does not depend on B


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 128])
@pytest.mark.parametrize("kind", [1, 2, 3, 4])
def test_act_jvp_matches_float64(gpu, k, kind):
  from compare_gan_b200 import tape
  rs = np.random.RandomState(k + kind)
  n, per = 5, 1000
  x = rs.standard_normal((n, per)).astype(np.float32)
  ref = x if kind in (1, 2) else {3: 1 / (1 + np.exp(-x)), 4: (np.tanh(x) + 1) / 2}[kind].astype(np.float32)
  t = rs.standard_normal((n * k, per)).astype(np.float32)
  with gpu.forward_mode(n, k):
    got = gpu.act_jvp(tape.DT(_dev(t)), tape.DT(_dev(ref)), kind, 0.2).cpu()
  r = np.repeat(ref.astype(np.float64), k, axis=0)
  d = {1: (r > 0) * 1.0, 2: np.where(r > 0, 1.0, 0.2), 3: r * (1 - r), 4: 0.5 * (1 - (2 * r - 1) ** 2)}[kind]
  want = t * d
  assert np.all(np.abs(got - want) <= 4e-7 * np.abs(want) + 1e-30), np.max(np.abs(got - want))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 128])
@pytest.mark.parametrize("cond", [False, True])
@pytest.mark.parametrize("relu", [False, True])
def test_bn_apply_jvp_matches_float64(gpu, k, cond, relu):
  from compare_gan_b200 import tape
  rs = np.random.RandomState(k + 2 * cond + relu)
  b, rps, c = 3, 16, 12
  x = rs.standard_normal((b * rps, c)).astype(np.float32)
  mv = np.concatenate([rs.standard_normal(c), rs.uniform(0.5, 2.0, c)]).astype(np.float32)
  gamma = rs.standard_normal((b, c) if cond else (c,)).astype(np.float32)
  beta = rs.standard_normal((b, c) if cond else (c,)).astype(np.float32)
  tx = rs.standard_normal((b * rps * k, c)).astype(np.float32)
  tg = rs.standard_normal((b * k, c)).astype(np.float32) if cond else None
  tb = rs.standard_normal((b * k, c)).astype(np.float32) if cond else None
  xd, mvd, gd, bd = (tape.DT(_dev(v)) for v in (x, mv, gamma, beta))
  y = tape.DT(torch.empty_like(xd.t))
  gpu._call("bn_apply", y.ptr, xd.ptr, b * rps, c, rps, mvd.ptr, 1e-3, gd.ptr, bd.ptr, int(cond), int(relu))
  with gpu.forward_mode(b, k):
    got = gpu.bn_apply_jvp(tape.DT(_dev(tx)), xd, mvd, 1e-3, gd, None if tg is None else tape.DT(_dev(tg)),
                           None if tb is None else tape.DT(_dev(tb)), cond, y if relu else None).cpu()
  m64 = mv.astype(np.float64)
  inv = 1 / np.sqrt(m64[c:] + np.float32(1e-3))
  xhat = ((x - m64[:c]) * inv).reshape(b, 1, rps, c)
  g = gamma.astype(np.float64).reshape((b, 1, 1, c) if cond else (1, 1, 1, c))
  want = tx.reshape(b, k, rps, c) * inv * g
  if cond:
    want = want + xhat * tg.reshape(b, k, 1, c) + tb.reshape(b, k, 1, c)
  if relu:
    want = want * (y.cpu().reshape(b, 1, rps, c) > 0)
  want = want.reshape(-1, c)
  scale = np.abs(tx.reshape(b, k, rps, c) * inv * g).reshape(-1, c) + 1e-6
  if cond:
    scale = scale + (np.abs(xhat * tg.reshape(b, k, 1, c)) + np.abs(tb.reshape(b, k, 1, c))).reshape(-1, c)
  assert np.all(np.abs(got - want) <= 1e-6 * scale), np.max(np.abs(got - want) / scale)


@pytest.mark.gpu
def test_mlp_three_ways_on_the_gpu(gpu):
  check_mlp_three_ways(gpu)
  check_linear_case(gpu)


# ---- 7. on the H100: generators ----

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GENERATORS))
def test_generator_tangents_match_the_float64_oracle(gpu, name):
  check_generator(gpu, name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["biggan_conditional", "resnet_cifar"])
def test_pass_primal_equals_generate_batch_and_leaves_g_unchanged(gpu, name):
  from compare_gan_b200 import eval_gan_lib
  from tests.gpu_util import make_pair
  arch, shape, kw, zd = GENERATORS[name]
  eng, _ = make_pair(arch, shape, 6, z_dim=zd, **kw)
  eng.flat_g["param"].t.add_(0.01 * torch.randn_like(eng.flat_g["param"].t))      # weights away from the init
  before = {k: v.t.clone() for k, v in eng.store.vars.items()}
  gpu.set_math_mode(1)
  z, labels = _jc()._draw_latents(eng, 6, np.random.RandomState(4))
  with _jc()._GeneratorPass(eng, tangent_rows=2 * zd) as run:      # three chunks of two samples
    imgs, _ = run(z, labels)
  assert gpu._RT["math_mode"] == 1
  after = {k: v.t for k, v in eng.store.vars.items()}
  for k in before:
    assert torch.equal(before[k], after[k]), k
  gpu.set_math_mode(0)
  ref = eval_gan_lib.generate_batch(eng, 6, np.random.RandomState(4))
  gpu.set_math_mode(1)
  for k in before:
    after[k].copy_(before[k])
  assert torch.equal(imgs.t, ref.t)
  gpu.set_math_mode(0)


@pytest.mark.gpu
@pytest.mark.parametrize("g_sn", [True, False])
def test_evaluation(gpu, g_sn):
  """FID / IS bit-identical with and without the task, count 64 and finite statistics; graph equal to eager for a G
  without spectral norm (its u advances on every G call, and the graph path calls G a different number of times)."""
  from compare_gan_b200 import eval_gan_lib
  from compare_gan_b200.metrics import fid_score, inception_score
  from tests.gpu_util import make_pair
  eng, _ = make_pair("resnet_biggan_arch", (32, 32, 3), 4, g_bn="conditional_batch_norm", g_sn=g_sn, conditional=True,
                     num_classes=10, z_dim=120, ch=8)
  n = 300
  real = np.random.RandomState(5).rand(n, 32, 32, 3).astype(np.float32)
  kw = dict(num_averaging_runs=2, num_samples=n, batch_size=32, seed=7, real_images=real)
  base = [inception_score.InceptionScoreTask(), fid_score.FIDScoreTask()]
  state = {k: v.t.clone() for k, v in eng.store.vars.items()}

  def run(tasks, use_graph):
    for k, v in eng.store.vars.items():
      v.t.copy_(state[k])
    return eval_gan_lib.evaluate(eng, tasks, use_graph=use_graph, **kw)
  res = run(base + [_jc().GeneratorConditionNumberTask()], True)
  without = run(base, True)
  for key in ("fid_score_mean", "fid_score_list", "inception_score_mean", "inception_score_list"):
    assert res[key] == without[key], key
  assert res["log_condition_number_count_mean"] == 64
  assert np.isfinite(res["log_condition_number_mean_mean"]) and np.isfinite(res["log_condition_number_std_mean"])
  if not g_sn:
    eager = run(base + [_jc().GeneratorConditionNumberTask()], False)
    for key in ("log_condition_number_mean_list", "log_condition_number_std_list"):
      assert res[key] == eager[key], key
