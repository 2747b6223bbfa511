/* cgan_b200.h — C-ABI of the H100 (sm_90a) GAN-step / FID engine.
 *
 * The reference (google/compare_gan) has no FFI: its seam is the Python ops library
 * (compare_gan/architectures/arch_ops.py, resnet_ops.py, gans/loss_lib.py, gans/penalty_lib.py,
 * tf.train.AdamOptimizer, tfgan FID).  Each entry point below replaces the TF library kernel(s)
 * behind one of those call sites; the citation after each declaration is the reference
 * file:line it stands in for (paths relative to the reference's compare_gan/ package).
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer unless named host_*.
 *  - activations float32 NHWC; conv kernels HWIO [kh,kw,cin,cout]; linear kernels [in,out]
 *    (arch_ops.py:543-546, 563-565, 583-585).
 *  - every call is asynchronous on the context's stream (cgan_ctx_set_stream); no call
 *    synchronises or allocates after warm-up (workspace grows on first use only).
 *  - return 0 on success, non-zero error code otherwise; message via cgan_last_error().
 *    Nothing throws across the ABI.  A context is not thread-safe.
 */
#ifndef CGAN_B200_H_
#define CGAN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cgan_ctx cgan_ctx;

enum { CGAN_OK = 0, CGAN_ERR_ARG = 1, CGAN_ERR_CUDA = 2, CGAN_ERR_WORKSPACE = 3, CGAN_ERR_UNSUPPORTED = 4 };

/* ---- context ------------------------------------------------------------------------- */
int cgan_version(void);
int cgan_ctx_create(cgan_ctx** out, int device);
int cgan_ctx_destroy(cgan_ctx* ctx);
int cgan_ctx_set_stream(cgan_ctx* ctx, void* cuda_stream);          /* cudaStream_t */
int cgan_ctx_reserve_workspace(cgan_ctx* ctx, size_t bytes);        /* pre-size (never during capture) */
/* 0: exact fp32 SIMT contraction; 1: wgmma TF32 tensor-core path where the shape allows. */
int cgan_ctx_set_math_mode(cgan_ctx* ctx, int mode);
const char* cgan_last_error(cgan_ctx* ctx);
/* number of kernels this context has launched since creation (bench.py's gpu_launches). */
int64_t cgan_launch_count(cgan_ctx* ctx);
/* Tuning knobs and introspection (tests compare kernel variants bit for bit and ask which path a contraction took).
 *   CGAN_OPT_TC_MT      (set/get) max pixel tiles (conv) / work units (filter gradient) per tensor-core CTA: 1 or 2
 *                       (2 only where it pays: convolution column tiles <= 64 wide, so that two CTAs still share an SM;
 *                       filter-gradient column tiles <= 128 wide, where the accumulators of both fit the registers).
 *   CGAN_OPT_TC_HALO    (set/get) 3x3 stride-1 tensor-core convolutions fetch one (rows+2)-row activation box per kernel
 *                       column instead of one box per tap: 0 never, 1 where the operand is rounded in the kernel and there
 *                       are >= 256 output channels (default), 2 wherever the geometry allows.
 *   CGAN_OPT_TC_THIN    (set/get) 1 (default): in math_mode 1 the image-side convolutions (<= 4 input or <= 4 output channels,
 *                       kh*kw*channels <= 32: every discriminator's first and every generator's last convolution, Inception's
 *                       stem) run as ONE 32-wide GEMM on the tensor-core kernels over a [pixels, 32] patch tensor (csrc/thin_tc.cu),
 *                       TF32 operands like every other tensor-core contraction; 0: the exact-fp32 streaming kernels (thin.cu).
 *   CGAN_OPT_LAST_PATH  (get) CGAN_PATH_* taken by the most recent conv2d_fwd / dgrad / wgrad / gemm / gemm_batched call.
 *   CGAN_OPT_LAST_TC_BN, CGAN_OPT_LAST_TC_MT, CGAN_OPT_LAST_TC_HALO
 *                       (get) column-tile width, pixel tiles per CTA and halo kernel (1) or per-tap kernel (0) of the most
 *                       recent tensor-core convolution kernel launch (the wgmma implicit GEMM, not the filter gradient);
 *                       0 before the first one.
 *   CGAN_OPT_LAST_TC_CTAS_PER_SM
 *                       (get) CTAs of that launch that fit on one SM at its dynamic shared memory, as the CUDA occupancy
 *                       calculator reports it; 0 before the first one.
 *   CGAN_OPT_LAST_TC_EP_SMEM
 *                       (get) 1 when that launch had its residual or ReLU mask prefetched into shared memory by TMA, 0
 *                       when its epilogue read them (if any) from global memory; 0 before the first one.
 *   CGAN_OPT_LAST_TC_TMA_STORE
 *                       (get) 1 when that launch staged its output tiles in shared memory and stored them by TMA, 0 when
 *                       its epilogue stored them from registers; 0 before the first one. */
enum { CGAN_OPT_TC_MT = 1, CGAN_OPT_LAST_PATH = 2, CGAN_OPT_TC_HALO = 3, CGAN_OPT_TC_THIN = 6, CGAN_OPT_LAST_TC_BN = 7,
       CGAN_OPT_LAST_TC_MT = 8, CGAN_OPT_LAST_TC_HALO = 9, CGAN_OPT_LAST_TC_CTAS_PER_SM = 10,
       CGAN_OPT_LAST_TC_EP_SMEM = 11, CGAN_OPT_LAST_TC_TMA_STORE = 12 };
/* CGAN_PATH_TCGEN05_TF32 keeps its name for ABI compatibility: the TF32 tensor-core (wgmma) path. */
enum { CGAN_PATH_SIMT_FP32 = 0, CGAN_PATH_TCGEN05_TF32 = 1, CGAN_PATH_THIN_FP32 = 2 };
int cgan_ctx_set_option(cgan_ctx* ctx, int key, int64_t value);
int cgan_ctx_get_option(cgan_ctx* ctx, int key, int64_t* host_value);

/* ---- utilities ------------------------------------------------------------------------ */
int cgan_fill(cgan_ctx*, float* dst, float value, int64_t n);
int cgan_copy(cgan_ctx*, float* dst, const float* src, int64_t n);
/* dst[r, dst_off + j] = src[r, src_off + j], j < cols  (tf.concat / tf.split on axis 1) */
int cgan_copy2d(cgan_ctx*, float* dst, int dst_ld, int dst_off, const float* src, int src_ld, int src_off,
                int64_t rows, int cols);
/* y = a*x + b*y0 + c   (y0 nullable) — x*2-1 (sndcgan.py:108), (tanh+1)/2, grad accumulation */
int cgan_axpby(cgan_ctx*, float* y, float a, const float* x, float b, const float* y0, float c, int64_t n);
/* y[i] = x[i] * (*scalar_dev) * mul  — non_local_block sigma (arch_ops.py:758), 1/sigma scaling */
int cgan_scale_by_dev(cgan_ctx*, float* y, const float* x, const float* scalar_dev, float mul, int inverse, int64_t n);
/* out[0] = sum_i a[i]*b[i]  (deterministic two-stage) — d sigma of non_local_block, SN backward */
int cgan_dot(cgan_ctx*, float* out_dev, const float* a, const float* b, int64_t n);
/* out[i] = uniform [0, 1) from the counter-based generator SplitMix64(seed, offset + i) (24 mantissa bits): the
 * tf.random.uniform draws of the gradient penalties (gans/penalty_lib.py:72-73) when the caller does not feed them.
 * Stateless: the same (seed, offset) always yields the same numbers, on any launch configuration. */
int cgan_random_uniform(cgan_ctx*, float* out, int64_t n, uint64_t seed, uint64_t offset);
/* y[n,:] = x[n,:] + alpha[n]*(xf[n,:]-x[n,:]) — WGAN-GP interpolates (gans/penalty_lib.py:74-75) */
int cgan_interpolate(cgan_ctx*, float* y, const float* x, const float* xf, const float* alpha, int n, int64_t per);
/* one-hot rows: out[n, labels[n]] = 1 (gans/modular_gan.py:359-363) */
int cgan_one_hot(cgan_ctx*, float* out, const int32_t* labels, int n, int classes);

/* ---- contractions ---------------------------------------------------------------------- */
typedef struct {
  int32_t n, h, w, cin;      /* real input tensor [n,h,w,cin] */
  int32_t cout, kh, kw, stride;
  int32_t upsample;          /* 1: input is zero-inserted 2x first (resnet_ops.py:35-56, :122-123), never materialised */
  int32_t oh, ow;            /* output spatial size */
  int32_t pad_t, pad_l;      /* TF SAME: before = total/2 */
} cgan_conv_desc;

/* y = conv(x, w) + bias   — tf.nn.conv2d(..., "SAME") + bias_add, arch_ops.py:568-572;
 * with desc.upsample: conv(unpool(x)), resnet_ops.py:122-130. */
int cgan_conv2d_fwd(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* w_hwio, const float* bias, float* y);
/* same with a fused activation (act = 0 or CGAN_ACT_RELU): conv + folded-BN bias + ReLU of the Inception graph
 * (tfgan.eval.run_inception, eval_utils.py:165-175); inference only. */
int cgan_conv2d_fwd_act(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* w_hwio, const float* bias, int act,
                        float* y);
/* same, writing output pixel p's `cout` channels at y + p*ldy (ldy >= cout): the convolution stores straight into its
 * channel slice of a wider NHWC tensor, which is tf.concat(axis=3) of the Inception "mixed" blocks without the copy
 * (tfgan.eval.run_inception, eval_utils.py:165-175).  Not available with desc.upsample. */
int cgan_conv2d_fwd_act_ld(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* w_hwio, const float* bias, int act,
                           float* y, int ldy);
/* dx = d/dx of the above (TF Conv2DBackpropInput); this is also tf.nn.conv2d_transpose, arch_ops.py:588-589. */
int cgan_conv2d_dgrad(cgan_ctx*, const cgan_conv_desc*, const float* dy, const float* w_hwio, float* dx);
/* dw = d/dw (TF Conv2DBackpropFilter); deterministic split-K. */
int cgan_conv2d_wgrad(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* dy, float* dw);
/* Fused forms of the three convolution entry points: what the reference writes as separate TF ops around a convolution
 * inside its residual blocks is done in the convolution's epilogue, so each activation tensor crosses HBM once:
 *   y = act(conv(x, w) + bias + residual)                 residual add of resnet_ops.py:181 / resnet_biggan.py:150
 *   act = ReLU when flags & CGAN_CONV_RELU                 tf.nn.relu of resnet_ops.py:161,174 (the consumer's pre-activation)
 *   y = pass ? y : mask_leak * y                           the (leaky-)ReLU gradient (arch_ops.py:595-597) applied to an input
 *                                                          gradient: mask is the activation's input (or output), same shape as y;
 *                                                          pass = mask >= 0 (-0 included) for leaky ReLU, mask > 0 for ReLU
 *   CGAN_CONV_ROUND_OUT: y is stored rounded to the nearest TF32 value (its only consumers are tensor-core contractions,
 *   which would round it anyway); CGAN_CONV_IN_TF32 / CGAN_CONV_IN2_TF32 assert that the first / second activation operand
 *   (x or dy; for wgrad x and dy) already holds TF32-representable values, so the kernel skips its operand-rounding pass.
 * In math_mode 0 (exact fp32) the rounding flags must not be set by the caller.  ldy: output pixel stride (0 = cout). */
enum { CGAN_CONV_RELU = 1, CGAN_CONV_ROUND_OUT = 2, CGAN_CONV_IN_TF32 = 4, CGAN_CONV_IN2_TF32 = 8 };
typedef struct {
  const float* bias;        /* [cout] (fwd) / [cin] (dgrad), nullable */
  const float* residual;    /* same shape as the output, nullable */
  const float* mask;        /* same shape as the output, nullable */
  float mask_leak;          /* 0 for ReLU, the leak for leaky ReLU (a leak of 0 means ReLU) */
  int32_t flags;
  int32_t ldy;
} cgan_conv_epilogue;
int cgan_conv2d_fwd_ex(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* w_hwio, const cgan_conv_epilogue* ep,
                       float* y);
int cgan_conv2d_dgrad_ex(cgan_ctx*, const cgan_conv_desc*, const float* dy, const float* w_hwio, const cgan_conv_epilogue* ep,
                         float* dx);
int cgan_conv2d_wgrad_ex(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* dy, int flags, float* dw);
/* C = alpha*op(A)*op(B) + beta*C, row-major, op = transpose when flag set — tf.matmul in
 * linear (arch_ops.py:548), projection head (resnet_biggan.py:419-423), attention (arch_ops.py:744,753). */
int cgan_gemm(cgan_ctx*, int trans_a, int trans_b, int m, int n, int k, float alpha, const float* a, int lda,
              const float* b, int ldb, float beta, float* c, int ldc);
int cgan_gemm_batched(cgan_ctx*, int trans_a, int trans_b, int m, int n, int k, float alpha, const float* a, int lda,
                      int64_t stride_a, const float* b, int ldb, int64_t stride_b, float beta, float* c, int ldc,
                      int64_t stride_c, int batch);

/* ---- fused self-attention (non_local_block, arch_ops.py:734-753) --------------------------------------------------
 * out[i] = softmax(q[i] k[i]^T) v[i] per image i: q = theta [batch, lq, dk], k = phi [batch, lk, dk], v = g [batch, lk, dv],
 * out [batch, lq, dv] — tf.matmul(theta, phi, transpose_b=True) -> tf.nn.softmax -> tf.matmul(attn, g) in ONE wgmma
 * kernel: the [lq, lk] scores live in registers only (csrc/attn_tc.cu).  lse [batch, lq] receives the
 * log-sum-exp of every score row; the backward recomputes the probabilities from it.  Operands are consumed as TF32:
 * pass tensors that already hold TF32-representable values (cgan_round_tf32, or a producer's ROUND_OUT epilogue).
 * cgan_attention_supported returns 1 when the fused kernels accept the shape in the current math mode (math_mode 1,
 * lq and lk multiples of 128, dk <= 32 and a multiple of 4, dv <= 128 and a multiple of 16), else 0 — callers then
 * compose cgan_gemm_batched / cgan_softmax_* as the reference does.  The kernels read q, k, v and dout as float4 and store
 * out, dq, dk, dv and read lse as float2: other pointers (legal 4-byte-aligned ones) return CGAN_ERR_UNSUPPORTED without
 * launching. */
int cgan_attention_supported(cgan_ctx*, int batch, int lq, int lk, int dk, int dv);
int cgan_attention_fwd(cgan_ctx*, const float* q, const float* k, const float* v, float* out, float* lse, int batch, int lq,
                       int lk, int dk, int dv);
/* gradients of the above w.r.t. q, k, v given dout [batch, lq, dv] (TF's MatMul / Softmax gradients of arch_ops.py:744-753):
 * two kernels, one accumulating dq per query tile, one accumulating dk and dv per key tile; fixed summation order. */
int cgan_attention_bwd(cgan_ctx*, const float* q, const float* k, const float* v, const float* out, const float* lse,
                       const float* dout, float* dq, float* dk_out, float* dv_out, int batch, int lq, int lk, int dk, int dv);
/* y = x rounded to the nearest TF32 value (10 mantissa bits), what a tensor-core contraction in math_mode 1 does to its operands */
int cgan_round_tf32(cgan_ctx*, float* y, const float* x, int64_t n);

/* ---- rows x channels reductions / bias -------------------------------------------------- */
/* y[r,c] = x[r,c] + bias[c]   (linear bias, arch_ops.py:549-555) */
int cgan_bias_add(cgan_ctx*, float* y, const float* x, const float* bias, int64_t rows, int c);
/* out[g,c] = sum over the rows of group g of x[r,c]; rows = groups*rows_per_group (bias / beta gradients) */
int cgan_colsum(cgan_ctx*, float* out, const float* x, int groups, int64_t rows_per_group, int c);

/* ---- batch norm (arch_ops.py:194-319, 327-367, 423-445; tpu/tpu_ops.py:94-125) ------------ */
/* local moments: mean[c] = sum x / rows, meansq[c] = sum x^2 / rows  (fp32; stats[0:c]=mean, stats[c:2c]=meansq).
 * Cross-replica BN all-reduces this [2c] buffer and divides by the replica count (tpu_ops.py:110-125). */
int cgan_bn_moments(cgan_ctx*, float* stats2c, const float* x, int64_t rows, int c);
/* var = meansq - mean^2 (arch_ops.py:289-297 / tpu_ops.py:125); optional moving-average update
 * m <- m - (m - batch)*(1-decay) (arch_ops.py:100-117); moving_* nullable. */
int cgan_bn_finalize(cgan_ctx*, float* mean_var2c, const float* stats2c, int c, float* moving_mean, float* moving_var,
                     float decay);
/* accumulator inference path (arch_ops.py:122-191): if *update_accus_dev==1 accumulate; write accu/counter to mean_var2c */
int cgan_bn_accumulate(cgan_ctx*, float* mean_var2c, const float* batch_mean_var2c, int c, float* accu_mean,
                       float* accu_var, float* accu_counter, const float* update_accus_dev);
/* y = (x-mean)*rsqrt(var+eps)*gamma + beta; gamma/beta: [c] (cond=0) or [samples,c] (cond=1, one row per sample of
 * rows_per_sample rows); either nullable; act: 0 none, 1 relu. */
int cgan_bn_apply(cgan_ctx*, float* y, const float* x, int64_t rows, int c, int64_t rows_per_sample,
                  const float* mean_var2c, float eps, const float* gamma, const float* beta, int cond, int act);
/* backward of training-mode BN.  Step 1 (reduce): sums2c[0:c] = sum dxhat, sums2c[c:2c] = sum dxhat*xhat over LOCAL rows
 * (all-reduced by the caller under cross-replica BN); dgamma/dbeta: [c] or [samples,c] (nullable). */
int cgan_bn_bwd_reduce(cgan_ctx*, float* sums2c, float* dgamma, float* dbeta, const float* dy, const float* x,
                       int64_t rows, int c, int64_t rows_per_sample, const float* mean_var2c, float eps,
                       const float* gamma, int cond);
/* Step 2: dx = inv*(dxhat - sums[0]/count - xhat*sums[1]/count), count = GLOBAL rows; round_tf32: store dx rounded to the
 * nearest TF32 value (it is the dy operand of the producing convolution's tensor-core gradients). */
int cgan_bn_bwd_apply(cgan_ctx*, float* dx, const float* dy, const float* x, int64_t rows, int c, int64_t rows_per_sample,
                      const float* mean_var2c, float eps, const float* gamma, int cond, const float* sums2c,
                      float inv_count, int round_tf32);

/* ---- self-modulated batch norm (arch_ops.py:370-420) -----------------------------------------------------------------
 * The MLP that turns z [n, z_dim] into one layer's scale and offset: h = relu(z w_h + b_h) [n, hidden] (h = z when
 * hidden = 0, the reference's num_hidden = 0), gamma = h w_gamma + b_gamma, beta = h w_beta + b_beta [n, c].  gb [2n, c]
 * holds gamma in rows 0..n-1 and beta in rows n..2n-1: each half is the [samples, c] gamma / beta of
 * cgan_bn_apply(cond = 1).  Weights are [in, out] as in linear.  K = hidden (or z_dim when hidden = 0) must be <= 256,
 * n <= 12288.  Exact fp32 in both math modes; every output is summed in a fixed order without atomics, so reruns and
 * graph replays are bit-identical.
 * Forward: one launch; writes gb and (hidden > 0) h, the post-ReLU hidden state the backward reads. */
int cgan_self_modulation_fwd(cgan_ctx*, float* gb, float* h, const float* z, int n, int z_dim, int hidden,
                             const float* w_h, const float* b_h, const float* w_gamma, const float* b_gamma,
                             const float* w_beta, const float* b_beta, int c);
/* Backward for the cotangent dgb [2n, c]: dw_gamma = h^T dgamma, db_gamma = sum dgamma (beta alike); dh = (dgamma
 * w_gamma^T + dbeta w_beta^T) * [h > 0], dw_h = z^T dh, db_h = sum dh, dz = dh w_h^T (dz = dh when hidden = 0).  Every
 * output is nullable (dw_h / db_h need hidden > 0).  One launch for the wide layer, a second for dh's cross-CTA sum when
 * dw_h, db_h or dz is asked for.  Workspace: per-CTA partials of dh, at most 64 MB. */
int cgan_self_modulation_bwd(cgan_ctx*, float* dw_h, float* db_h, float* dw_gamma, float* db_gamma, float* dw_beta,
                             float* db_beta, float* dz, const float* dgb, const float* h, const float* z,
                             const float* w_h, const float* w_gamma, const float* w_beta, int n, int z_dim, int hidden,
                             int c);
/* Forward-mode tangent (biases and weights constant): t_z [n * k, z_dim] sample-major as cgan_act_jvp's batches,
 * t_h = (t_z w_h) * [h[s] > 0] for the rows of sample s (t_h = t_z when hidden = 0), t_gb [2n * k, c] = t_h w_gamma in
 * rows 0..nk-1 and t_h w_beta in rows nk..2nk-1: the t_gamma / t_beta halves cgan_bn_apply_jvp takes.  One launch. */
int cgan_self_modulation_jvp(cgan_ctx*, float* t_gb, const float* t_z, const float* h, const float* w_h,
                             const float* w_gamma, const float* w_beta, int n, int z_dim, int hidden, int c, int k);

/* ---- layer norm (arch_ops.py:448-450: tf.contrib.layers.layer_norm, begin_norm_axis=1, begin_params_axis=-1) -------
 * x is [n, span] with span = h*w*c (NHWC samples): the moments of sample i run over its whole span, gamma and beta are
 * [c].  stats2n[2i] = mean, stats2n[2i+1] = r = rsqrt(var + eps) (contrib's float32 eps is 1e-12).  Each span is split over
 * several CTAs; their float64 partials are merged in a fixed order (Chan et al.'s pairwise update), so results are
 * deterministic.  Workspace through the context; no host synchronisation (capturable). */
int cgan_layer_norm_moments(cgan_ctx*, float* stats2n, const float* x, int n, int64_t span, float eps);
/* y = (x - mean) * (r * gamma) + beta; act: 0 none, 1 ReLU, optionally | CGAN_ACT_ROUND_TF32 */
int cgan_layer_norm_apply(cgan_ctx*, float* y, const float* x, int n, int64_t span, int c, const float* stats2n,
                          const float* gamma, const float* beta, int act);
/* backward for the cotangent g on y: dx = r * (a - mean(a) - xhat * mean(a*xhat)) with a = gamma*g, xhat = (x - mean)*r,
 * means per sample; dgamma = sum g*xhat, dbeta = sum g over all pixels.  dx, dgamma, dbeta nullable; round_tf32: store
 * dx rounded to the nearest TF32 value. */
int cgan_layer_norm_bwd(cgan_ctx*, float* dx, float* dgamma, float* dbeta, const float* g, const float* x, int n,
                        int64_t span, int c, const float* stats2n, const float* gamma, int round_tf32);
/* double backward: the vjp of (g, x, gamma) -> dx above for the cotangent w on dx.  With P(w) = w - mean(w) -
 * xhat*mean(w*xhat): d_g = gamma * r * P(w), d_gamma = sum over pixels of g * r * P(w), and d_x is the vjp of TF's graph,
 * whose variance reads stop_gradient(mean): the exact d_x minus r^2 * mean(a*xhat) * mean(w) per sample.  Outputs
 * nullable; round_tf32 applies to d_x. */
int cgan_layer_norm_bwd_bwd(cgan_ctx*, float* d_g, float* d_x, float* d_gamma, const float* w, const float* g,
                            const float* x, int n, int64_t span, int c, const float* stats2n, const float* gamma,
                            int round_tf32);

/* ---- DRAGAN and L2 penalties (penalty_lib.py:33-57, 85-103) ------------------------------------------------------ */
/* DRAGAN's perturbed real batch (penalty_lib.py:47-50): y = clip(x + std * (U - 0.5), 0, 1) over the n floats of x, with
 * var the float64 variance of all n elements rounded once to fp32 (the layer-norm moments of one sample spanning the
 * batch), std = sqrtf(var), and U[i] = cgan_random_uniform's element at (seed, offset = step * n + i), step read from the
 * device counter step_dev (the discriminator's Adam step before its update).  Each operation rounds on its own.  std is
 * also written to the device scalar std_out.  Two launches, no host synchronisation (capturable; replays draw at the
 * counter's new value). */
int cgan_dragan_perturb(cgan_ctx*, float* y, const float* x, int64_t n, uint64_t seed, const int32_t* step_dev,
                        float* std_out);
/* L2 penalty over the kernels of a packed parameter buffer (penalty_lib.py:98-102): segs_dev holds nseg (offset, length)
 * pairs in floats; out[0] = mean over segments of sum(w^2) / 2, squared and summed in float64 in an order fixed by the
 * table alone, rounded once to fp32.  One launch. */
int cgan_l2_penalty(cgan_ctx*, float* out, const float* flat_param, const int64_t* segs_dev, int nseg);
/* its gradient: flat_grad[j] += fp32(fp32(scale_dev[0] * mul) * flat_param[j]) for every j inside a segment; nothing
 * else is touched.  One launch. */
int cgan_l2_penalty_bwd(cgan_ctx*, float* flat_grad, const float* flat_param, const int64_t* segs_dev, int nseg,
                        const float* scale_dev, float mul);

/* ---- spectral norm (arch_ops.py:453-535) -------------------------------------------------- */
/* One power iteration on w[rows,cols]; left=1: u[rows], v[cols] (arch_ops.py:505-509,525); left=0: u[cols], v[rows]
 * (:511-513,527).  u is updated in place (:516); v and sigma are outputs; wbar = w / sigma (nullable). */
int cgan_spectral_norm(cgan_ctx*, const float* w, int rows, int cols, int left, float eps, float* u_inout, float* v_out,
                       float* sigma_out, float* wbar_out);
/* The same for `n` weights in ONE launch (one CTA per weight; meant for the small kernels of a discriminator — resnet_cifar,
 * SNDCGAN — where the per-weight entry point costs ~7 launches each).  `items_dev` is a device array; item i reads w / u,
 * updates u in place and writes wbar at wbar_base + wbar_off, v at v_base + v_off, sigma at sigma_base[i] and a copy of
 * the updated u (which the backward needs; later call sites overwrite u) at u_used_base + u_off.
 * max_rows_plus_cols = max over items of rows + cols (shared-memory sizing). */
typedef struct {
  const float* w;
  float* u;
  int32_t rows, cols, left, reserved;
  int64_t wbar_off, v_off, u_off;
} cgan_sn_item;
int cgan_spectral_norm_batched(cgan_ctx*, const cgan_sn_item* items_dev, int n, int max_rows_plus_cols, float eps,
                               float* wbar_base, float* v_base, float* sigma_base, float* u_used_base);
/* dw = (dwbar - <dwbar, wbar> * outer) / sigma, outer = u v^T (left) or v u^T (right); u,v constants (:521-522). */
int cgan_spectral_norm_bwd(cgan_ctx*, float* dw, const float* dwbar, const float* wbar, int rows, int cols, int left,
                           const float* u, const float* v, const float* sigma);

/* ---- pointwise / pooling ------------------------------------------------------------------- */
enum { CGAN_ACT_RELU = 1, CGAN_ACT_LRELU = 2, CGAN_ACT_SIGMOID = 3, CGAN_ACT_TANH01 = 4 /* (tanh(x)+1)/2 */ };
/* OR-ed into `kind` (act_fwd / act_bwd) or `act` (bn_apply): store the result rounded to the nearest TF32 value — the
 * tensor only feeds tensor-core contractions, which then skip their own operand-rounding pass (math_mode 1 only). */
enum { CGAN_ACT_ROUND_TF32 = 0x100 };
int cgan_act_fwd(cgan_ctx*, float* y, const float* x, int kind, float leak, int64_t n);
/* dx = dy * act'(.) ; `ref` is x for relu/lrelu and y for sigmoid/tanh01.  TF's rule at 0: relu' = [ref > 0] (ReluGrad),
 * lrelu' = 1 where ref >= 0, -0 included (tf.maximum(x, leak x) sends a tie's gradient to x), else leak. */
int cgan_act_bwd(cgan_ctx*, float* dx, const float* dy, const float* ref, int kind, float leak, int64_t n);
int cgan_add(cgan_ctx*, float* y, const float* a, const float* b, int64_t n);
/* same, optionally storing TF32-rounded sums (gradient accumulation in front of a tensor-core contraction) */
int cgan_add_tf32(cgan_ctx*, float* y, const float* a, const float* b, int64_t n, int round_tf32);
/* 2x2 stride-2 average pool (resnet_ops.py:131-133) and its adjoint */
int cgan_avgpool2_fwd(cgan_ctx*, float* y, const float* x, int n, int h, int w, int c);
int cgan_avgpool2_bwd(cgan_ctx*, float* dx, const float* dy, int n, int h, int w, int c);
/* 2x2 stride-2 max pool (arch_ops.py:741,750) and backward (first-max wins, as TF MaxPoolGrad) */
int cgan_maxpool2_fwd(cgan_ctx*, float* y, const float* x, int n, int h, int w, int c);
int cgan_maxpool2_bwd(cgan_ctx*, float* dx, const float* dy, const float* x, int n, int h, int w, int c);
/* generic k x k pooling, TF semantics: mode 0 = max, 1 = average that EXCLUDES padded cells from the divisor (tf.nn.avg_pool
 * "SAME"); pad_t/pad_l = leading padding (0 for "VALID"); oh/ow given by the caller.  Inception-v3 feature extractor
 * (tfgan.eval.run_inception, eval_utils.py:165-175). */
int cgan_pool2d_fwd(cgan_ctx*, float* y, const float* x, int n, int h, int w, int c, int k, int stride, int pad_t, int pad_l,
                    int oh, int ow, int mode);
/* global pool over h*w: out[n,c] = scale * sum_hw x (mean: resnet_cifar.py:156; sum: resnet_biggan.py:405) */
int cgan_globalpool_fwd(cgan_ctx*, float* y, const float* x, int n, int hw, int c, float scale);
int cgan_globalpool_bwd(cgan_ctx*, float* dx, const float* dy, int n, int hw, int c, float scale);
/* row softmax (tf.nn.softmax, arch_ops.py:745) and its backward */
int cgan_softmax_fwd(cgan_ctx*, float* y, const float* x, int64_t rows, int cols);
int cgan_softmax_bwd(cgan_ctx*, float* dx, const float* dy, const float* y, int64_t rows, int cols);
/* out[r] = sum_j a[r,j]*b[r,j]  (projection discriminator, resnet_biggan.py:423) */
int cgan_rowdot(cgan_ctx*, float* out, const float* a, const float* b, int64_t rows, int cols);
/* y[r,j] = a[r,j] * s[r] */
int cgan_rowscale(cgan_ctx*, float* y, const float* a, const float* s, int64_t rows, int cols);

/* ---- losses and penalties ------------------------------------------------------------------ */
enum { CGAN_LOSS_NON_SATURATING = 0, CGAN_LOSS_HINGE = 1, CGAN_LOSS_WASSERSTEIN = 2, CGAN_LOSS_LEAST_SQUARES = 3 };
/* gans/loss_lib.py:53-148.  out4 = {d_loss, d_loss_real, d_loss_fake, g_loss}.  dlogits[2b] (nullable) receives
 * d(d_loss)/dlogit (which=0) or d(g_loss)/dlogit (which=1) for the [real; fake] logit vector. */
int cgan_gan_loss(cgan_ctx*, int kind, const float* logits_real, const float* logits_fake, int b, float* out4,
                  float* dlogits, int which);
/* gans/penalty_lib.py:78-81: slopes = sqrt(1e-4 + sum_hwc g^2); penalty = mean((slopes-1)^2);
 * dg (nullable) = d(weight*penalty)/dg. */
int cgan_gp_penalty(cgan_ctx*, float* penalty_out, float* dg, const float* g, int n, int64_t per, float weight);

/* ---- self-supervision (gans/ssgan.py, gans/utils.py:38-49) ------------------------------------------------------ */
/* y = x rotated by k * 90 degrees (k = 1, 2, 3), square NHWC images: rotate_images' transposes / flips in one pass. */
int cgan_rot90(cgan_ctx*, float* y, const float* x, int n, int hw, int c, int k);
/* rotation loss: `rows` = num_rotations * m logit rows [rows, num_rotations], row r labelled r / m;
 * *loss_out = -mean log(softmax(logits)[label] + 1e-10) (ssgan.py:205-213); dlogits (nullable) = its gradient. */
int cgan_rotation_loss(cgan_ctx*, float* loss_out, float* dlogits, const float* logits, int rows, int num_rotations);

/* ---- S3GAN heads (gans/s3gan.py) --------------------------------------------------------------------------------------
 * out[r] = 1 if sum_j y[r, j] > 0.5 else 0: "is a label available for this example" (s3gan.py:121-122). */
int cgan_row_has_label(cgan_ctx*, float* out, const float* y, int rows, int cols);
/* out[r, :] = one_hot(argmax_j logits[r, j]) (first maximum wins, like tf.argmax): the predictor's hard labels
 * (s3gan.py:149-150). */
int cgan_argmax_one_hot(cgan_ctx*, float* out, const float* logits, int rows, int cols);
/* tf.losses.softmax_cross_entropy(onehot_labels = labels, logits, weights) with its default SUM_BY_NONZERO_WEIGHTS reduction
 * (s3gan.py:312-313): *loss_out = sum_r w_r * (-sum_j labels[r,j] log softmax(logits_r)_j) / max(#{w_r != 0}, 1); labels may
 * be soft; weights [rows] nullable (= 1).  dlogits (nullable) receives d loss / d logits. */
int cgan_softmax_xent(cgan_ctx*, float* loss_out, float* dlogits, const float* logits, const float* labels,
                      const float* weights, int rows, int cols);

/* ---- optimizer (tf.train.AdamOptimizer + tf.train.ExponentialMovingAverage, gans/modular_gan.py:498-508) ---- */
/* One fused multi-tensor step over a flat parameter buffer.  *step_dev (int32, device) is incremented first; then
 * lr_t = lr*sqrt(1-b2^t)/(1-b1^t); m,v updated; p -= lr_t*m/(sqrt(v)+eps).  If ema != NULL:
 * ema <- ema - (ema-p)*(1-d), d = ema_decay*[ (t-1) >= ema_start_step ]. grad_scale multiplies g first (1/world). */
int cgan_adam_step(cgan_ctx*, float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2,
                   float eps, float grad_scale, int32_t* step_dev, float* ema, float ema_decay, int32_t ema_start_step);

/* ---- FID statistics (tfgan frechet_classifier_distance_from_activations, metrics/fid_score.py:49-51) ---- */
/* sum[d] += sum_n act[n,d]; sumxxT[d,d] += act^T act, accumulated in float64 on device. */
int cgan_cov_accumulate(cgan_ctx*, const float* act, int n, int d, double* sum, double* sumxxT);
/* bilinear resize NHWC [n,h,w,c] -> [n,oh,ow,c] (tf.image.resize_bilinear, align_corners=False) then (x*255-128)/128
 * when `inception_scale` (eval_utils.py:157-175). */
int cgan_resize_bilinear(cgan_ctx*, float* y, const float* x, int n, int h, int w, int c, int oh, int ow, int inception_scale);

/* ---- data set transforms (ImageNet / CelebA / LSUN input transforms, datasets.py:374-427, 440-532) ---- */
/* One element of a packed uint8 batch (cgan_loader_next_packed).  Its window, h x w pixels of c channels HWC, starts
 * `offset` bytes into the packed batch and sits on a canvas_h x canvas_w canvas with its top-left pixel at (top, left);
 * canvas pixels outside the window are 0 (tf.image.resize_image_with_crop_or_pad's padding).  position is the element's
 * place p in the repeated stream, element its source index, (crop_y, crop_x) the window's origin in the source image. */
typedef struct cgan_crop_desc {
  int64_t offset;
  int64_t position;
  int32_t element;
  int32_t h, w;
  int32_t canvas_h, canvas_w;
  int32_t top, left;
  int32_t crop_y, crop_x;
  int32_t reserved;
} cgan_crop_desc;
/* out [n, r, r, c] fp32 NHWC: each element's canvas resized to r x r by TF1's legacy bilinear resize
 * (tf.image.resize_images: align_corners = False, src = dst * (in / out), no half-pixel offset), every operation a
 * separately rounded fp32 operation (no FMA contraction).  divide_after = 0 divides each uint8 tap by 255 before the
 * interpolation (ImageNet: tf.cast / 255, then resize), 1 interpolates the uint8 values and divides the result by 255
 * (CelebA: resize, then / 255); both are true divisions.  packed: device bytes of the batch, desc [n] device descriptors
 * (their offsets count from `packed`); c is 1 or 3. */
int cgan_crop_resize_u8(cgan_ctx*, float* out, const uint8_t* packed, const cgan_crop_desc* desc, int n, int c, int r,
                        int divide_after);

/* ---- MS-SSIM terms (metrics/image_similarity.py:85-211, 239-333) ---- */
/* Per-scale SSIM terms of image pairs of ONE image set.  images [n,h,w,c] fp32 NHWC, values in [0, max_val];
 * host_pairs [npairs,2] int32 HOST indices into the set (they travel to the device in the kernel parameters, so the call
 * stays asynchronous and capturable); out [npairs, levels, c] fp32: the mean over output pixels of cs for levels
 * 0..levels-2 and of luminance*cs for the last level, before the relu.  Level l is level l-1 average-pooled 2x2 after
 * repeating its last row / column where a side is odd; its window is the Gaussian of width filter_width and size
 * min(filter_size, level height, level width) (<= 64), applied VALID.  Requires h, w >= 2^(levels-1), levels <= 16.
 * A pair's bits do not depend on the other pairs of the call; (i, j) and (j, i) give the same bits; identical images
 * give exactly 1.  The host finishes MS-SSIM (relu, power factors, product over levels, mean over channels). */
int cgan_ssim_terms(cgan_ctx*, float* out, const float* images, int n, int h, int w, int c, const int32_t* host_pairs,
                    int npairs, int levels, int filter_size, float filter_width, float max_val);

/* ---- k-means of the PRD histograms (metrics/prd_score.py:94-122, the MiniBatchKMeans fit of _cluster_into_bins) ---- */
/* `groups` independent clusterings of the same points x [m,d] fp32 into k clusters (1 <= k <= 64, m >= k), in float64
 * throughout: squared distances ||x||^2 + ||c||^2 - 2 x.c with x.c on the FP64 tensor cores (DMMA), the nearest centre
 * being the first minimum.  Centroids are [groups, k, d] float64.  A group's results do not depend on the other groups of
 * the call, and reruns are bit-identical.
 *
 * k-means++ seeding: host_uniforms [groups, k] float64 HOST values in [0, 1) (checked on the host, then copied to the
 * workspace).  Centre 0 of group g is point min(floor(u[g,0] m), m-1); centre j is the smallest i with
 * cumsum(w)[i] > u[g,j] * cumsum(w)[m-1], cumsum a sequential float64 sum and w[i] = max(0, squared distance of point i
 * to its nearest chosen centre); when cumsum(w)[m-1] == 0, point min(floor(u m), m-1). */
int cgan_kmeans_seed(cgan_ctx*, double* centroids, const float* x, int m, int d, int k, int groups,
                     const double* host_uniforms);
/* One Lloyd iteration (sklearn KMeans(algorithm="lloyd")) of every group whose state[g,0] is 0: assign every point to
 * its nearest centre (labels [groups, m] int32), then move each centre to the float64 mean of its points (summed in
 * point order; an EMPTY cluster keeps its centre).  state [groups, 2] int32, zero before the first step:
 * (status, iterations done); status becomes 2 when the labels equal those of the group's previous step, else 1 when the
 * total squared centre shift is <= tol, and stays 0 otherwise.  Finished groups cost nothing.  The caller reads state
 * back to decide whether to step again (max_iter is the caller's). */
int cgan_kmeans_lloyd_step(cgan_ctx*, double* centroids, int32_t* labels, int32_t* state, const float* x, int m, int d,
                           int k, int groups, double tol);
/* Final assignment against the given centroids: labels [groups, m] int32, inertia [groups] float64 (the sum of the
 * squared distances in a fixed order), counts [groups, 2, k] int32: the points of each cluster among rows [0, n_eval)
 * and among rows [n_eval, m). */
int cgan_kmeans_finish(cgan_ctx*, int32_t* labels, double* inertia, int32_t* counts, const double* centroids,
                       const float* x, int m, int d, int k, int groups, int n_eval);

/* ---- fractal dimension (metrics/fractal_dimension.py:39-97) ---- */
/* out [n, s] float64: out[i, j] = sqrt(sum_k (x'[i, k] - s'[j, k])^2) with x' = fp32(scale * x[i, k]) and
 * s' = fp32(scale * seeds[j, k]) (x [n, d], seeds [s, d] fp32; scale = 255 gives the reference's float32 images * 255,
 * eval_utils.py:157), each converted to float64 before the subtraction, the squares accumulated with a float64 FMA and
 * the sqrt correctly rounded: the scipy.spatial.distance.cdist of fractal_dimension.py:67-68.  Direct differences, so
 * a row equal to a seed is at distance exactly 0.  A row's bits depend on d only: not on n, on the other rows of the
 * call or on the call's position in a run.  Workspace: partial sums of D slices, at most 64 MB. */
int cgan_fd_distances(cgan_ctx*, double* out, const float* x, int n, const float* seeds, int s, int d, float scale);
/* out2[0] = the smallest non-zero and out2[1] = the largest of dist[0, count) (non-negative values), exact
 * (fractal_dimension.py:69-70); out2[0] = +inf when every value is 0, and out2[1] is NaN when one is. */
int cgan_fd_range(cgan_ctx*, double* out2, const double* dist, int64_t count);
/* counts[j] = #{q < count : dist[q] < edges[j]} for non-decreasing edges [nedges] in device memory (1 <= nedges <= 8192):
 * np.sum(np.less.outer(dist, edges), axis=0) of fractal_dimension.py:78, exact (integer histogram + prefix sum). */
int cgan_fd_counts(cgan_ctx*, int64_t* counts, const double* dist, int64_t count, const double* edges, int nedges);

/* ---- generator conditioning (metrics/jacobian_conditioning.py:32-173) ---- */
/* Forward-mode tangents of the generator's nonlinear ops.  A tangent batch holds k tangents per primal sample,
 * sample-major: for n_primal samples of `per` values each, t[(s * k + j) * per + e] is tangent j of value e of sample s,
 * and the primal (ref / x / y / p) is read once per tangent: t_out = t_in * act'(ref), with ref = x for relu / lrelu (1 where
 * ref > 0, else 0 / 1 where ref >= 0, else leak) and ref = y for sigmoid / tanh01, as cgan_act_bwd (arch_ops.py:595-597, sndcgan.py:74-78). */
int cgan_act_jvp(cgan_ctx*, float* t_out, const float* t_in, const float* ref, int kind, float leak, int n_primal,
                 int64_t per, int k);
/* Tangent of cgan_bn_apply with the moments constant (arch_ops.py:66-191, 423-445): r = rsqrt(var + eps),
 * xhat = (x - mean) r, t_y = t_x r gamma + xhat t_gamma + t_beta, then zero where y <= 0 when y (the primal output of a
 * fused ReLU) is given.  x [rows, c] primal, rows_per_sample rows per sample; t_x / t_y [rows * k, c]; gamma [c]
 * (cond = 0) or [rows / rows_per_sample, c] (cond = 1), nullable; t_gamma / t_beta [rows / rows_per_sample * k, c],
 * cond = 1 only, nullable; t_x nullable (a zero tangent). */
int cgan_bn_apply_jvp(cgan_ctx*, float* t_y, const float* t_x, const float* x, const float* y, int64_t rows, int c,
                      int64_t rows_per_sample, const float* mean_var2c, float eps, const float* gamma, const float* t_gamma,
                      const float* t_beta, int cond, int k);
/* Tangent of cgan_maxpool2_fwd (arch_ops.py:741, 750): the tangent at the first maximum of the primal window. */
int cgan_maxpool2_jvp(cgan_ctx*, float* t_out, const float* t_in, const float* x, int n_primal, int h, int w, int c, int k);
/* Tangent of cgan_softmax_fwd (arch_ops.py:745): t_out = p (t_in - <t_in, p>) per row, which is cgan_softmax_bwd with
 * the primal probabilities p [n_primal * rows_per_sample, cols] broadcast over the k tangents of each sample. */
int cgan_softmax_jvp(cgan_ctx*, float* t_out, const float* t_in, const float* p, int n_primal, int64_t rows_per_sample,
                     int cols, int k);
/* Metric tensors M[b] = T[b] T[b]^T (jacobian_conditioning.py:146-173; there a float32 np.matmul) in float64: T [B, k, D]
 * fp32 (the tangent output of B samples, k tangents each), M [B, k, k] float64.  The fp32 values are converted exactly,
 * products are formed on the FP64 tensor cores and summed over fixed D slices in a fixed order: reruns are
 * bit-identical, a sample's result does not depend on B, and M[b] is exactly symmetric.  Workspace: slice sums, at most
 * 64 MB (or one sample's). */
int cgan_metric_tensor_f64(cgan_ctx*, double* M, const float* T, int B, int k, int64_t D);

/* ---- cross-replica exchange of small vectors (tpu/tpu_ops.py:75-125: cross_replica_mean / cross_replica_moments) ---- */
/* One process per GPU on one node.  Every rank allocates a communication buffer and publishes its cudaIpc handle
 * (cgan_p2p_local_handle -> 64 bytes), the host code all-gathers the handles (torch.distributed) and hands all of them
 * to cgan_p2p_connect, which maps the peers' buffers.  cgan_allreduce_small then sums x[0..n) over the ranks IN PLACE
 * with one kernel launch over NVLink peer memory (n <= cgan_p2p_max_floats()): every rank stores its vector into every
 * peer's buffer, flags it, waits for the others' flags and adds the vectors in rank order — bit-identical results on all
 * ranks, capturable into a CUDA graph.  Gradients (MBs) stay on NCCL (gans/modular_gan.py:606-616). */
int cgan_p2p_max_floats(void);
int cgan_p2p_local_handle(cgan_ctx*, int world, void* host_handle64);
int cgan_p2p_connect(cgan_ctx*, int rank, int world, const void* host_handles);
int cgan_allreduce_small(cgan_ctx*, float* x, int n);

/* ---- input pipeline (ImageDatasetV2.train_input_fn, datasets.py:261-291; host side, no GPU work) ---- */
/* The tf.data chain of the reference: repeat() -> shuffle(buffer, seed) -> batch(drop_remainder=True) -> prefetch, with
 * _parse_fn's uint8 -> float32 / 255 (datasets.py:225-227), run by a producer thread into a ring of `ring` batch buffers
 * (page-locked when a CUDA device is present, so the caller's cudaMemcpyAsync overlaps the previous step).
 * Source: `n` images NHWC contiguous in host memory, uint8 (src_dtype 0, scaled by 1/255) or float32 (src_dtype 1, copied;
 * the reference's fake data set, datasets.py:136-145), and optional int32 labels; caller-owned, must outlive the loader
 * (e.g. an mmap of a shard file).  shuffle_buffer <= 1 disables shuffling.  The shuffle is tf.data's algorithm (a buffer
 * of `shuffle_buffer` elements, each output drawn uniformly from it and replaced by the next input) on a SplitMix64
 * stream; the element ORDER is therefore not TF's (its Philox stream is not restated). */
typedef struct cgan_loader cgan_loader;
int cgan_loader_create(cgan_loader** out, const void* images, int src_dtype, const int32_t* labels, int64_t n, int h, int w,
                       int c, int batch, int shuffle_buffer, uint64_t seed, int ring);
/* Blocks until the next batch is ready: images float32 [batch,h,w,c], labels int32 [batch] (zeros without source
 * labels).  The buffers stay untouched until released; with every ring slot outstanding the call fails instead of
 * dead-locking. */
int cgan_loader_next(cgan_loader*, const float** images, const int32_t** labels);
/* Hands the `count` oldest outstanding batches back to the producer (call once their host->device copies finished). */
int cgan_loader_release(cgan_loader*, int count);
int cgan_loader_destroy(cgan_loader*);
const char* cgan_loader_last_error(cgan_loader*);

/* Sources of any image size for the transformed path: n images of c channels, image i being index[i] = (offset, h, w)
 * row-major HWC uint8 at pixels + offset (host memory, caller-owned, must outlive the loader), and optional int32
 * labels. */
typedef struct cgan_image_source {
  const uint8_t* pixels;
  int64_t pixel_bytes;
  const int64_t* index;
  const int32_t* labels;
  int64_t n;
  int32_t c;
  int32_t reserved;
} cgan_image_source;
enum { CGAN_CROP_NONE = 0, CGAN_CROP_MIDDLE = 1, CGAN_CROP_RANDOM = 2, CGAN_CROP_DISTORTED = 3, CGAN_CROP_OR_PAD = 4 };
enum { CGAN_LABEL_SOURCE = 0, CGAN_LABEL_ZERO = 1, CGAN_LABEL_RANDOM = 2 };
/* The per-element transform (datasets.py:374-427, 440-584).  crop: CGAN_CROP_* (datasets.py:458-491; CGAN_CROP_OR_PAD is
 * tf.image.resize_image_with_crop_or_pad to canvas_h x canvas_w).  Filters, applied once at creation (an empty element
 * list is an error): min_side > 0 keeps images with min(h, w) >= min_side, labeled_only keeps labels >= 0.  label:
 * CGAN_LABEL_SOURCE (0 without source labels), CGAN_LABEL_ZERO, or CGAN_LABEL_RANDOM (uniform in [0, random_classes),
 * drawn anew for every stream position). */
typedef struct cgan_image_transform {
  int32_t crop;
  int32_t canvas_h, canvas_w;
  int32_t min_side;
  int32_t labeled_only;
  int32_t label;
  int32_t random_classes;
  int32_t reserved;
} cgan_image_transform;
/* A loader whose producer packs, per element, only the rows of the element's crop window: each ring slot holds the
 * batch's cgan_crop_desc table ([batch] descriptors at the start of the slot) followed by the packed window bytes, ready
 * for ONE host->device copy and cgan_crop_resize_u8.  The element of stream position p is list[p % n] (list: the filtered
 * source indices, in source order); the shuffle is cgan_loader_create's.  Random crops and labels are keyed by
 * (seed, p, draw index) through SplitMix64, so they depend on neither the shuffle buffer nor thread timing. */
int cgan_loader_create_transformed(cgan_loader** out, const cgan_image_source* source, const cgan_image_transform* transform,
                                   int batch, int shuffle_buffer, uint64_t seed, int ring);
/* cgan_loader_next for a transformed loader: *slot_data points at the slot ([batch] descriptors, then the packed bytes),
 * *slot_bytes is the size of what the batch used, labels int32 [batch]. */
int cgan_loader_next_packed(cgan_loader*, const uint8_t** slot_data, int64_t* slot_bytes, const int32_t** labels);

#ifdef __cplusplus
}
#endif
#endif  /* CGAN_B200_H_ */
