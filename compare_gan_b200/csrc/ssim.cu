// Per-scale SSIM terms of image pairs: the O(pixels) part of MS-SSIM (metrics/image_similarity.py:85-211, 239-333).
//
// The reference tiles a batch into all ordered pairs and runs five 2-D depthwise convolutions per pair and scale.  Here:
//   - every level of every image's pyramid is built once, planar and shifted by max_val / 2 (x' = x - max_val / 2, which
//     keeps the second moments small: the covariance is a difference of them);
//   - the per-image maps mu' = G * x' and v = G * x'^2 - mu'^2 are filtered once per image (G: the Gaussian window, applied
//     separably: the reference's 2-D softmax window is the outer product of two normalised 1-D Gaussians);
//   - only G * (x' y') is filtered per pair; luminance and contrast-structure are then evaluated per output pixel.
// The shift cancels algebraically: cov = G * (x' y') - mu'_x mu'_y and var = G * x'^2 - mu'^2; the luminance uses
// mu = mu' + max_val / 2.
//
// Exactness: each filtered value is summed in a fixed tap order by the same device code in both passes, so a pair of
// identical images has G * (x' y') == G * x'^2 bit for bit and the products / sums below are formed without contraction:
// luminance and cs are then exactly 1 (as the literal fp32 formula gives).  Every operation is commutative in (x, y), so
// (i, j) and (j, i) give the same bits.  One CTA owns one (pair, channel) and sums its pixels in a fixed order: a pair's
// result does not depend on the other pairs of the call.
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int SS_MAX_LEVELS = 16, SS_MAX_WIN = 64;
constexpr int SS_CHUNK = 1024;          // pairs per launch; the indices travel in the kernel parameters
constexpr int SS_TH = 16, SS_TW = 64;   // output tile of the separable filter; 256 threads
constexpr int SS_THREADS = 256;

struct SsimGeom {
  int n, c, levels;
  int h[SS_MAX_LEVELS], w[SS_MAX_LEVELS], f[SS_MAX_LEVELS], oh[SS_MAX_LEVELS], ow[SS_MAX_LEVELS];
  long long pyr_off[SS_MAX_LEVELS];     // floats: level l of the pyramid, planar [n, c, h, w]
  long long map_off[SS_MAX_LEVELS];     // float2s: (mu', v) of level l, planar [n, c, oh, ow]
  float win[SS_MAX_LEVELS][SS_MAX_WIN]; // normalised 1-D Gaussian of width f[l]
  float shift, c1, c2;
};

struct SsimPairs {
  int2 p[SS_CHUNK];
};

__host__ __device__ inline int ss_in_stride(int f) { return (SS_TH + f - 1) | 1; }   // odd: conflict-free columns
__host__ __device__ inline size_t ss_smem_floats(int f) {
  return (size_t)(SS_TW + f - 1) * ss_in_stride(f) + (size_t)(SS_TH + f - 1) * (SS_TW + 1) + SS_MAX_WIN;
}

// Filters one SS_TH x SS_TW output tile at (r0, c0) of a (h, w) plane: the operand is a (PRODUCT = 0) or a * b.
// Leaves four vertically adjacent outputs in out[0..3]: rows r0 + 4 * (tid / SS_TW) + j, column c0 + tid % SS_TW.
// s_in holds the input tile column-major, s_hz the horizontally filtered rows.
template <int PRODUCT>
__device__ __forceinline__ void ss_filter_tile(const float* __restrict__ a, const float* __restrict__ b, int h, int w, int f,
                                               int r0, int c0, const float* win, float* s_in, float* s_hz, float out[4]) {
  const int ih = SS_TH + f - 1, iw = SS_TW + f - 1, ihp = ss_in_stride(f);
  for (int e = threadIdx.x; e < ih * iw; e += SS_THREADS) {
    const int r = e / iw, cc = e - r * iw, gr = r0 + r, gc = c0 + cc;
    float v = 0.f;
    if (gr < h && gc < w) {
      const long long o = (long long)gr * w + gc;
      v = PRODUCT ? __fmul_rn(a[o], b[o]) : a[o];
    }
    s_in[cc * ihp + r] = v;
  }
  __syncthreads();
  // horizontal: row r, columns 4g .. 4g + 3, sliding over the taps
  for (int e = threadIdx.x; e < ih * (SS_TW / 4); e += SS_THREADS) {
    const int r = e % ih, oc = 4 * (e / ih);
    const float* p = s_in + oc * ihp + r;
    float v0 = p[0], v1 = p[ihp], v2 = p[2 * ihp];
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int k = 0; k < f; ++k) {
      const float v3 = p[(k + 3) * ihp], wk = win[k];
      a0 = fmaf(wk, v0, a0); a1 = fmaf(wk, v1, a1); a2 = fmaf(wk, v2, a2); a3 = fmaf(wk, v3, a3);
      v0 = v1; v1 = v2; v2 = v3;
    }
    float* q = s_hz + r * (SS_TW + 1) + oc;
    q[0] = a0; q[1] = a1; q[2] = a2; q[3] = a3;
  }
  __syncthreads();
  // vertical: column tid % SS_TW, rows 4 * (tid / SS_TW) .. + 3
  {
    const int oc = threadIdx.x % SS_TW, or0 = 4 * (threadIdx.x / SS_TW);
    const float* p = s_hz + or0 * (SS_TW + 1) + oc;
    float v0 = p[0], v1 = p[SS_TW + 1], v2 = p[2 * (SS_TW + 1)];
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int k = 0; k < f; ++k) {
      const float v3 = p[(k + 3) * (SS_TW + 1)], wk = win[k];
      a0 = fmaf(wk, v0, a0); a1 = fmaf(wk, v1, a1); a2 = fmaf(wk, v2, a2); a3 = fmaf(wk, v3, a3);
      v0 = v1; v1 = v2; v2 = v3;
    }
    out[0] = a0; out[1] = a1; out[2] = a2; out[3] = a3;
  }
  __syncthreads();   // s_in / s_hz are reused by the next tile
}

// level 0 of the pyramid: NHWC images -> planar [n, c, h, w], shifted
__global__ void ssim_planar_kernel(float* __restrict__ y, const float* __restrict__ x, int n, int h, int w, int c, float shift) {
  const long long tot = (long long)n * h * w * c;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (long long)gridDim.x * blockDim.x) {
    const int ch = (int)(i % c);
    const long long pix = i / c, img = pix / ((long long)h * w), hw = pix - img * h * w;
    y[(img * c + ch) * h * w + hw] = __fsub_rn(x[i], shift);
  }
}

// level l from level l - 1 (planar planes of hi x wi): 2x2 average pool, VALID, after repeating the last row / column
// where a side is odd (tf.pad SYMMETRIC by one at the end, image_similarity.py:284-310)
__global__ void ssim_pool_kernel(float* __restrict__ y, const float* __restrict__ x, long long planes, int hi, int wi) {
  const int ho = (hi + 1) / 2, wo = (wi + 1) / 2;
  const long long tot = planes * ho * wo;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % wo);
    const long long t = i / wo;
    const int oy = (int)(t % ho);
    const long long pl = t / ho;
    const int y0 = 2 * oy, y1 = min(2 * oy + 1, hi - 1), x0 = 2 * ox, x1 = min(2 * ox + 1, wi - 1);
    const float* p = x + pl * hi * wi;
    const float s = (p[(long long)y0 * wi + x0] + p[(long long)y0 * wi + x1]) + (p[(long long)y1 * wi + x0] + p[(long long)y1 * wi + x1]);
    y[i] = s * 0.25f;
  }
}

__device__ __forceinline__ void ss_load_win(const SsimGeom& g, int l, float* s_win) {
  for (int k = threadIdx.x; k < g.f[l]; k += SS_THREADS) s_win[k] = g.win[l][k];
  __syncthreads();
}

// per-image maps (mu', v) of every level: grid (n * c, levels)
__global__ void __launch_bounds__(SS_THREADS) ssim_moments_kernel(const __grid_constant__ SsimGeom g, float* __restrict__ ws) {
  extern __shared__ float ss_smem[];
  const int plane = blockIdx.x, l = blockIdx.y;
  const int h = g.h[l], w = g.w[l], f = g.f[l], oh = g.oh[l], ow = g.ow[l];
  float* s_win = ss_smem;
  float* s_in = s_win + SS_MAX_WIN;
  float* s_hz = s_in + (size_t)(SS_TW + f - 1) * ss_in_stride(f);
  ss_load_win(g, l, s_win);
  const float* x = ws + g.pyr_off[l] + (long long)plane * h * w;
  float2* maps = reinterpret_cast<float2*>(ws) + g.map_off[l] + (long long)plane * oh * ow;
  const int oc = threadIdx.x % SS_TW, or0 = 4 * (threadIdx.x / SS_TW);
  for (int r0 = 0; r0 < oh; r0 += SS_TH)
    for (int c0 = 0; c0 < ow; c0 += SS_TW) {
      float mu[4], sq[4];
      ss_filter_tile<0>(x, x, h, w, f, r0, c0, s_win, s_in, s_hz, mu);
      ss_filter_tile<1>(x, x, h, w, f, r0, c0, s_win, s_in, s_hz, sq);
      const int col = c0 + oc;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int row = r0 + or0 + j;
        if (row < oh && col < ow) maps[(long long)row * ow + col] = make_float2(mu[j], __fsub_rn(sq[j], __fmul_rn(mu[j], mu[j])));
      }
    }
}

// out[(pair * levels + l) * c + ch] for the chunk's pairs: grid (pairs in chunk, c)
__global__ void __launch_bounds__(SS_THREADS) ssim_pairs_kernel(const __grid_constant__ SsimGeom g,
                                                                const __grid_constant__ SsimPairs pr, const float* __restrict__ ws,
                                                                float* __restrict__ out) {
  extern __shared__ float ss_smem[];
  __shared__ double red[SS_THREADS];
  const int ch = blockIdx.y, c = g.c, levels = g.levels;
  const int2 ij = pr.p[blockIdx.x];
  const int oc = threadIdx.x % SS_TW, or0 = 4 * (threadIdx.x / SS_TW);
  const float shift = g.shift, c1 = g.c1, c2 = g.c2;
  for (int l = 0; l < levels; ++l) {
    const int h = g.h[l], w = g.w[l], f = g.f[l], oh = g.oh[l], ow = g.ow[l];
    float* s_win = ss_smem;
    float* s_in = s_win + SS_MAX_WIN;
    float* s_hz = s_in + (size_t)(SS_TW + f - 1) * ss_in_stride(f);
    ss_load_win(g, l, s_win);
    const long long pi = (long long)ij.x * c + ch, pj = (long long)ij.y * c + ch;
    const float* x = ws + g.pyr_off[l] + pi * h * w;
    const float* y = ws + g.pyr_off[l] + pj * h * w;
    const float2* mx = reinterpret_cast<const float2*>(ws) + g.map_off[l] + pi * oh * ow;
    const float2* my = reinterpret_cast<const float2*>(ws) + g.map_off[l] + pj * oh * ow;
    const bool last = l == levels - 1;
    double acc = 0.0;
    for (int r0 = 0; r0 < oh; r0 += SS_TH)
      for (int c0 = 0; c0 < ow; c0 += SS_TW) {
        float pxy[4];
        ss_filter_tile<1>(x, y, h, w, f, r0, c0, s_win, s_in, s_hz, pxy);
        const int col = c0 + oc;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int row = r0 + or0 + j;
          if (row >= oh || col >= ow) continue;
          const long long o = (long long)row * ow + col;
          const float2 a = mx[o], b = my[o];
          // cs = (2 cov + c2) / (var_x + var_y + c2), cov = G*(x'y') - mu'_x mu'_y  (image_similarity.py:131-134)
          const float cov = __fsub_rn(pxy[j], __fmul_rn(a.x, b.x));
          const float cs = __fdiv_rn(__fadd_rn(__fmul_rn(2.f, cov), c2), __fadd_rn(__fadd_rn(a.y, b.y), c2));
          float term = cs;
          if (last) {   // luminance (2 mu_x mu_y + c1) / (mu_x^2 + mu_y^2 + c1) on the unshifted means (:120-124)
            const float ux = __fadd_rn(a.x, shift), uy = __fadd_rn(b.x, shift);
            const float num0 = __fmul_rn(2.f, __fmul_rn(ux, uy));
            const float den0 = __fadd_rn(__fmul_rn(ux, ux), __fmul_rn(uy, uy));
            term = __fmul_rn(__fdiv_rn(__fadd_rn(num0, c1), __fadd_rn(den0, c1)), cs);
          }
          acc += (double)term;
        }
      }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = SS_THREADS / 2; s > 0; s >>= 1) {
      if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x == 0) out[((long long)blockIdx.x * levels + l) * c + ch] = (float)(red[0] / ((double)oh * ow));
    __syncthreads();
  }
}

}  // namespace

int cgan_ssim_terms(cgan_ctx* ctx, float* out, const float* images, int n, int h, int w, int c, const int32_t* host_pairs,
                    int npairs, int levels, int filter_size, float filter_width, float max_val) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, out && images && host_pairs, "null pointer");
  CGAN_REQUIRE(ctx, n >= 1 && h >= 1 && w >= 1 && c >= 1 && npairs >= 1, "empty image set or pair list");
  CGAN_REQUIRE(ctx, levels >= 1 && levels <= SS_MAX_LEVELS, "levels must be in [1, 16]");
  CGAN_REQUIRE(ctx, filter_size >= 1 && filter_width > 0.f && max_val > 0.f, "filter_size, filter_width and max_val must be positive");
  CGAN_REQUIRE(ctx, (h >> (levels - 1)) >= 1 && (w >> (levels - 1)) >= 1, "image too small for levels - 1 halvings");
  CGAN_REQUIRE(ctx, filter_size <= SS_MAX_WIN || (h <= SS_MAX_WIN || w <= SS_MAX_WIN), "window (min(filter_size, h, w)) larger than 64");
  for (int p = 0; p < 2 * npairs; ++p)
    CGAN_REQUIRE(ctx, host_pairs[p] >= 0 && host_pairs[p] < n, "pair index out of range");

  SsimGeom g;
  memset(&g, 0, sizeof(g));
  g.n = n; g.c = c; g.levels = levels;
  g.shift = 0.5f * max_val;
  g.c1 = (float)((0.01 * max_val) * (0.01 * max_val));
  g.c2 = (float)((0.03 * max_val) * (0.03 * max_val));
  long long pyr = 0, maps = 0;
  for (int l = 0; l < levels; ++l) {
    g.h[l] = l ? (g.h[l - 1] + 1) / 2 : h;
    g.w[l] = l ? (g.w[l - 1] + 1) / 2 : w;
    const int f = g.f[l] = std::min(filter_size, std::min(g.h[l], g.w[l]));   // image_similarity.py:185-189
    g.oh[l] = g.h[l] - f + 1;
    g.ow[l] = g.w[l] - f + 1;
    g.pyr_off[l] = pyr;
    pyr += ((long long)n * c * g.h[l] * g.w[l] + 3) / 4 * 4;
    g.map_off[l] = maps;
    maps += (long long)n * c * g.oh[l] * g.ow[l];
    // 1-D factor of f_special_gauss (image_similarity.py:140-154): exp(-(k - (f-1)/2)^2 / (2 sigma^2)), normalised
    double e[SS_MAX_WIN], sum = 0.0;
    for (int k = 0; k < f; ++k) {
      const double t = k - (f - 1) / 2.0;
      e[k] = exp(-0.5 * t * t / ((double)filter_width * filter_width));
      sum += e[k];
    }
    for (int k = 0; k < f; ++k) g.win[l][k] = (float)(e[k] / sum);
  }
  // workspace: the pyramid (floats) then the maps (float2, 8-byte aligned since pyr is a multiple of 4 floats)
  void* wsp = nullptr;
  const size_t bytes = (size_t)pyr * sizeof(float) + (size_t)maps * sizeof(float2);
  int rc = cgan_ws(ctx, bytes, &wsp);
  if (rc) return rc;
  float* ws = static_cast<float*>(wsp);
  for (int l = 0; l < levels; ++l) g.map_off[l] += pyr / 2;

  ssim_planar_kernel<<<ew_grid(ctx, (long long)n * h * w * c), 256, 0, ctx->stream>>>(ws, images, n, h, w, c, g.shift);
  CGAN_LAUNCHED(ctx);
  for (int l = 1; l < levels; ++l) {
    ssim_pool_kernel<<<ew_grid(ctx, (long long)n * c * g.h[l] * g.w[l]), 256, 0, ctx->stream>>>(
        ws + g.pyr_off[l], ws + g.pyr_off[l - 1], (long long)n * c, g.h[l - 1], g.w[l - 1]);
    CGAN_LAUNCHED(ctx);
  }
  const size_t smem = ss_smem_floats(g.f[0]) * sizeof(float);   // f[0] is the largest window
  CGAN_CUDA(ctx, cudaFuncSetAttribute(ssim_moments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CGAN_CUDA(ctx, cudaFuncSetAttribute(ssim_pairs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ssim_moments_kernel<<<dim3(n * c, levels), SS_THREADS, smem, ctx->stream>>>(g, ws);
  CGAN_LAUNCHED(ctx);
  for (int p0 = 0; p0 < npairs; p0 += SS_CHUNK) {
    const int cnt = std::min(SS_CHUNK, npairs - p0);
    SsimPairs pr;
    for (int i = 0; i < cnt; ++i) pr.p[i] = make_int2(host_pairs[2 * (p0 + i)], host_pairs[2 * (p0 + i) + 1]);
    ssim_pairs_kernel<<<dim3(cnt, c), SS_THREADS, smem, ctx->stream>>>(g, pr, ws, out + (long long)p0 * levels * c);
    CGAN_LAUNCHED(ctx);
  }
  return CGAN_OK;
}
