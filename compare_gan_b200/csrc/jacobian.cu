// Generator conditioning (metrics/jacobian_conditioning.py:32-173): forward-mode tangents of the generator's nonlinear
// ops and the float64 metric tensors M = J^T J of its Jacobians.
//
// A tangent batch holds k tangents per primal sample, sample-major: tangent row block b * k + j belongs to primal sample
// b.  The nonlinear ops read the primal value of a sample once per tangent row (the primal is broadcast over k); the
// linear ops need no kernel of their own (the caller runs the primal op's kernel on the tangent batch).
//
// mt_gram_kernel forms M[b] = T[b] T[b]^T for the fp32 tangent output T[b] [k, D] on the FP64 tensor cores
// (mma.sync m8n8k4 f64): the fp32 values are converted to float64 as they are staged in shared memory (exact), so every
// product is exact and only the float64 sums round.  D is cut into fixed slices of MT_SLICE columns, each summed in
// column order by one CTA, and the slice sums are added in slice order: the result does not depend on the launch
// configuration, and reruns are bit-identical.  Only the tiles on and below the diagonal are computed; the reduce pass
// writes element (i, j), i >= j, to both (i, j) and (j, i), so M is exactly symmetric.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int MT_BM = 64, MT_BK = 32, MT_THREADS = 128;
constexpr int MT_LDS = MT_BK + 4;                 // smem row stride (doubles), as km_dist_kernel's
constexpr int MT_SLICE = 2048;                    // D columns per slice: a multiple of MT_BK
constexpr long long MT_PART_BYTES = 64ll << 20;   // slice sums of one launch at most

static_assert(MT_SLICE % MT_BK == 0, "a slice holds whole k stages");

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// primal index of element i of a tangent batch: `per` values per sample, k tangents per sample
__device__ __forceinline__ long long primal_index(long long i, long long per, int k) {
  const long long s = i / ((long long)k * per);
  return s * per + i % per;
}

__device__ __forceinline__ float act_deriv(float r, int kind, float leak) {
  if (kind == CGAN_ACT_RELU) return r > 0.f ? 1.f : 0.f;
  if (kind == CGAN_ACT_LRELU) return relu_gate(r, 1.f, leak);   // as act_bwd: ties (x = +-0) go to x
  if (kind == CGAN_ACT_SIGMOID) return r * (1.0f - r);
  const float t = 2.0f * r - 1.0f;       // y = (tanh + 1) / 2  ->  tanh = 2y - 1
  return 0.5f * (1.0f - t * t);
}

__global__ void act_jvp_kernel(float* __restrict__ t_out, const float* __restrict__ t_in, const float* __restrict__ ref,
                               int kind, float leak, long long total, long long per, int k) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x)
    t_out[i] = t_in[i] * act_deriv(ref[primal_index(i, per, k)], kind, leak);
}

// t_y = t_x * r * gamma + xhat * t_gamma + t_beta, masked by y > 0 when relu; r, xhat as bn_apply_kernel computes them
__global__ void bn_apply_jvp_kernel(float* __restrict__ t_y, const float* __restrict__ t_x, const float* __restrict__ x,
                                    const float* __restrict__ y, long long total, int C, long long rows_per_sample,
                                    const float* __restrict__ mean_var, float eps, const float* __restrict__ gamma,
                                    const float* __restrict__ t_gamma, const float* __restrict__ t_beta, int cond, int k) {
  const long long per = rows_per_sample * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long p = primal_index(i, per, k);
    const long long trow = i / per;                       // tangent row block: sample * k + j
    const long long s = trow / k;
    const float inv = 1.0f / sqrtf(mean_var[C + c] + eps);
    const float g = gamma ? gamma[cond ? s * C + c : c] : 1.0f;
    float v = t_x ? t_x[i] * inv * g : 0.f;
    if (t_gamma) v += (x[p] - mean_var[c]) * inv * t_gamma[trow * C + c];
    if (t_beta) v += t_beta[trow * C + c];
    if (y && !(y[p] > 0.f)) v = 0.f;
    t_y[i] = v;
  }
}

// the tangent at the window position maxpool2_bwd routes the gradient to (the first maximum)
__global__ void maxpool2_jvp_kernel(float* __restrict__ t_out, const float* __restrict__ t_in, const float* __restrict__ x,
                                    long long total, int h, int w, int c, int k) {
  const int oh = h / 2, ow = w / 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % c);
    long long t = i / c;
    const int ox = (int)(t % ow);
    t /= ow;
    const int oy = (int)(t % oh);
    const long long img = t / oh;                          // tangent image: sample * k + j
    const long long pimg = img / k;
    const long long off = ((long long)(2 * oy) * w + 2 * ox) * c + ch;
    const long long offs[4] = {0, c, (long long)w * c, (long long)w * c + c};
    const float* xp = x + pimg * h * w * c + off;
    int best = 0;
    float bv = xp[0];
#pragma unroll
    for (int q = 1; q < 4; ++q)
      if (xp[offs[q]] > bv) {
        bv = xp[offs[q]];
        best = q;
      }
    t_out[i] = t_in[img * h * w * c + off + offs[best]];
  }
}

// t_out = p * (t_in - <t_in, p>) per row, p broadcast over the k tangents of its sample: one block per tangent row
__global__ void softmax_jvp_kernel(float* __restrict__ t_out, const float* __restrict__ t_in, const float* __restrict__ p,
                                   long long rows_per_sample, int cols, int k) {
  __shared__ float sh[32];
  const long long row = blockIdx.x;
  const long long prow = (row / (k * rows_per_sample)) * rows_per_sample + row % rows_per_sample;
  const float* tr = t_in + row * cols;
  const float* pr = p + prow * cols;
  float s = 0.f;
  for (int j = threadIdx.x; j < cols; j += blockDim.x) s += tr[j] * pr[j];
  s = block_sum(s, sh);
  for (int j = threadIdx.x; j < cols; j += blockDim.x) t_out[row * cols + j] = pr[j] * (tr[j] - s);
}

// grid (lower-triangle tiles, slices, samples); 4 warps as 2 x 2, each 32 x 32 = 4 x 4 DMMA tiles.
// part[(z * nb + b) * k * k + i * k + j] = sum over slice z of T[b, i, :] T[b, j, :] for the tile's (i, j).
__global__ void __launch_bounds__(MT_THREADS) mt_gram_kernel(double* __restrict__ part, const float* __restrict__ T,
                                                             int k, int d, int nb) {
  __shared__ double As[MT_BM * MT_LDS];
  __shared__ double Bs[MT_BM * MT_LDS];
  // tile t of the lower triangle: row block ti, column block tj <= ti
  int ti = 0, t = blockIdx.x;
  while (t > ti) {
    t -= ti + 1;
    ++ti;
  }
  const int tj = t;
  const int b = blockIdx.z;
  const int i0 = ti * MT_BM, j0 = tj * MT_BM;
  const int k_lo = blockIdx.y * MT_SLICE, k_hi = min(d, k_lo + MT_SLICE);
  const float* Tb = T + (long long)b * k * d;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp & 1, wn = warp >> 1;

  // staging: thread t loads column t % 32 of rows t / 32 + 4 r
  const int kc = tid & 31, r0 = tid >> 5;
  float ra[MT_BM / 4], rb[MT_BM / 4];
  auto load = [&](int k0) {
    const int col = k0 + kc;
#pragma unroll
    for (int r = 0; r < MT_BM / 4; ++r) {
      const int i = i0 + r0 + 4 * r, j = j0 + r0 + 4 * r;
      ra[r] = (i < k && col < k_hi) ? __ldg(Tb + (long long)i * d + col) : 0.f;
      rb[r] = (j < k && col < k_hi) ? __ldg(Tb + (long long)j * d + col) : 0.f;
    }
  };
  auto store = [&]() {
#pragma unroll
    for (int r = 0; r < MT_BM / 4; ++r) {
      As[(r0 + 4 * r) * MT_LDS + kc] = (double)ra[r];
      Bs[(r0 + 4 * r) * MT_LDS + kc] = (double)rb[r];
    }
  };

  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[a][q][0] = acc[a][q][1] = 0.0;

  const int fr = lane >> 2, fc = lane & 3;
  load(k_lo);
  for (int k0 = k_lo; k0 < k_hi; k0 += MT_BK) {
    __syncthreads();
    store();
    __syncthreads();
    if (k0 + MT_BK < k_hi) load(k0 + MT_BK);
#pragma unroll
    for (int kq = 0; kq < MT_BK; kq += 4) {
      double af[4], bf[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        af[q] = As[(wm * 32 + q * 8 + fr) * MT_LDS + kq + fc];
        bf[q] = Bs[(wn * 32 + q * 8 + fr) * MT_LDS + kq + fc];
      }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int q = 0; q < 4; ++q) dmma(acc[a][q][0], acc[a][q][1], af[a], bf[q]);
    }
  }

  double* out = part + ((long long)blockIdx.y * nb + b) * k * k;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int i = i0 + wm * 32 + a * 8 + fr;
    if (i >= k) continue;
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int j = j0 + wn * 32 + q * 8 + 2 * fc + h;
        if (j <= i) out[(long long)i * k + j] = acc[a][q][h];
      }
  }
}

// M[b, i, j] = M[b, j, i] = part[0, b, i, j] + part[1, b, i, j] + ..., i >= j, added in slice order
__global__ void mt_reduce_kernel(double* __restrict__ M, const double* __restrict__ part, int k, int nb, int nslices) {
  const long long kk = (long long)k * k, count = (long long)nb * kk;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < count; q += (long long)gridDim.x * blockDim.x) {
    const long long b = q / kk;
    const int i = (int)((q % kk) / k), j = (int)(q % k);
    if (j > i) continue;
    double v = part[q];
    for (int z = 1; z < nslices; ++z) v = __dadd_rn(v, part[(long long)z * count + q]);
    M[b * kk + (long long)i * k + j] = v;
    M[b * kk + (long long)j * k + i] = v;
  }
}

}  // namespace

int cgan_act_jvp(cgan_ctx* ctx, float* t_out, const float* t_in, const float* ref, int kind, float leak, int n_primal,
                 int64_t per, int k) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, t_out && t_in && ref, "null pointer");
  CGAN_REQUIRE(ctx, kind >= CGAN_ACT_RELU && kind <= CGAN_ACT_TANH01, "kind must be a CGAN_ACT_* activation");
  CGAN_REQUIRE(ctx, n_primal >= 1 && per >= 1 && k >= 1, "n_primal, per and k must be >= 1");
  const long long total = (long long)n_primal * k * per;
  act_jvp_kernel<<<ew_grid(ctx, total), 256, 0, ctx->stream>>>(t_out, t_in, ref, kind, leak, total, per, k);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_bn_apply_jvp(cgan_ctx* ctx, float* t_y, const float* t_x, const float* x, const float* y, int64_t rows, int c,
                      int64_t rows_per_sample, const float* mean_var2c, float eps, const float* gamma, const float* t_gamma,
                      const float* t_beta, int cond, int k) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, t_y && x && mean_var2c, "null pointer");
  CGAN_REQUIRE(ctx, rows >= 1 && c >= 1 && k >= 1 && rows_per_sample >= 1 && rows % rows_per_sample == 0,
               "rows, c, k >= 1 and rows_per_sample must divide rows");
  CGAN_REQUIRE(ctx, cond || (!t_gamma && !t_beta), "t_gamma / t_beta need cond = 1");
  CGAN_REQUIRE(ctx, !t_gamma || gamma, "t_gamma needs gamma");
  const long long total = (long long)rows * c * k;
  bn_apply_jvp_kernel<<<ew_grid(ctx, total), 256, 0, ctx->stream>>>(t_y, t_x, x, y, total, c, rows_per_sample, mean_var2c,
                                                                   eps, gamma, t_gamma, t_beta, cond, k);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_maxpool2_jvp(cgan_ctx* ctx, float* t_out, const float* t_in, const float* x, int n_primal, int h, int w, int c,
                      int k) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, t_out && t_in && x, "null pointer");
  CGAN_REQUIRE(ctx, n_primal >= 1 && h >= 2 && w >= 2 && c >= 1 && k >= 1, "bad shape");
  const long long total = (long long)n_primal * k * (h / 2) * (w / 2) * c;
  maxpool2_jvp_kernel<<<ew_grid(ctx, total), 256, 0, ctx->stream>>>(t_out, t_in, x, total, h, w, c, k);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_softmax_jvp(cgan_ctx* ctx, float* t_out, const float* t_in, const float* p, int n_primal, int64_t rows_per_sample,
                     int cols, int k) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, t_out && t_in && p, "null pointer");
  CGAN_REQUIRE(ctx, n_primal >= 1 && rows_per_sample >= 1 && cols >= 1 && k >= 1, "bad shape");
  const long long rows = (long long)n_primal * k * rows_per_sample;
  CGAN_REQUIRE(ctx, rows < (1ll << 31), "too many rows");
  softmax_jvp_kernel<<<(unsigned)rows, 256, 0, ctx->stream>>>(t_out, t_in, p, rows_per_sample, cols, k);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_metric_tensor_f64(cgan_ctx* ctx, double* M, const float* T, int B, int k, int64_t D) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, M && T, "null pointer");
  CGAN_REQUIRE(ctx, B >= 1 && k >= 1 && D >= 1, "B, k and D must be >= 1");
  CGAN_REQUIRE(ctx, k <= 4096 && D < (1ll << 31) && cdiv(D, MT_SLICE) <= 65535, "k <= 4096 and D < 2^31");
  const int nslices = cdiv(D, MT_SLICE);
  const int kb = cdiv(k, MT_BM), tiles = kb * (kb + 1) / 2;
  const long long per_sample = (long long)nslices * k * k * (long long)sizeof(double);
  long long nb = MT_PART_BYTES / per_sample;
  nb = nb < 1 ? 1 : (nb > B ? B : (nb > 65535 ? 65535 : nb));
  void* ws = nullptr;
  int rc = cgan_ws(ctx, (size_t)(nb * per_sample), &ws);
  if (rc) return rc;
  double* part = static_cast<double*>(ws);
  for (long long b0 = 0; b0 < B; b0 += nb) {
    const int n = (int)(B - b0 < nb ? B - b0 : nb);
    mt_gram_kernel<<<dim3(tiles, nslices, n), MT_THREADS, 0, ctx->stream>>>(part, T + b0 * k * D, k, (int)D, n);
    CGAN_LAUNCHED(ctx);
    mt_reduce_kernel<<<ew_grid(ctx, (long long)n * k * k), 256, 0, ctx->stream>>>(M + b0 * k * k, part, k, n, nslices);
    CGAN_LAUNCHED(ctx);
  }
  return CGAN_OK;
}
