// Batch-norm family (moments / apply / backward, conditional and cross-replica aware) and the
// spectral-norm power iteration.  All HBM-bound rows x channels work over NHWC activations:
// channels are the fastest dimension, so a warp reads 128 contiguous bytes of one row and the
// per-channel sums are reduced over row lanes in shared memory, then over chunks in a second,
// fixed-order (deterministic) pass.
//
// Replaces: standardize_batch (arch_ops.py:194-319), batch_norm (:327-367), conditional_batch_norm
// (:423-445), cross_replica_moments (tpu/tpu_ops.py:94-125), spectral_norm (arch_ops.py:453-535).
#include "common.cuh"

namespace {

constexpr int CR_X = 32, CR_Y = 8;   // column-reduce block: 32 channels x 8 row lanes

struct MomentsF {
  const float* x;
  __device__ __forceinline__ void operator()(long long r, int c, int C, long long, float* v) const {
    float t = x[r * C + c];
    v[0] = t;
    v[1] = t * t;
  }
};
struct SumF {
  const float* x;
  __device__ __forceinline__ void operator()(long long r, int c, int C, long long, float* v) const {
    v[0] = x[r * C + c];
  }
};
struct WeightedSumF {   // sum_r a[r] * w[r,c]  (W^T a)
  const float* w;
  const float* a;
  __device__ __forceinline__ void operator()(long long r, int c, int C, long long, float* v) const {
    v[0] = w[r * C + c] * a[r];
  }
};
struct BnBwdF {         // v0 = sum dy*xhat, v1 = sum dy
  const float* dy;
  const float* x;
  const float* mean_var;
  float eps;
  __device__ __forceinline__ void operator()(long long r, int c, int C, long long, float* v) const {
    float inv = 1.0f / sqrtf(mean_var[C + c] + eps);
    float xh = (x[r * C + c] - mean_var[c]) * inv;
    float g = dy[r * C + c];
    v[0] = g * xh;
    v[1] = g;
  }
};

// partial[((g*chunks + chunk)*NV + v)*C + c].  With `counters` the LAST chunk-block of each (column block, group) to finish
// also does the second stage — the fixed-order sum over the chunk partials that colreduce_final_kernel otherwise does in a
// launch of its own (same order, same result): every block publishes its partials (threadfence), takes a ticket, and the
// holder of ticket chunks-1 reads them all back.  The counter is reset by that block, so launches (and graph replays)
// always start from zero.
template <class F, int NV>
__global__ void colreduce_kernel(F f, float* __restrict__ partial, long long rows_per_group, int C,
                                 long long rows_per_chunk, int chunks, unsigned* counters, float scale, float* out0, float* out1) {
  __shared__ float sh[NV][CR_Y][CR_X + 1];
  __shared__ unsigned s_ticket;
  const int c = blockIdx.x * CR_X + threadIdx.x;
  const int chunk = blockIdx.y, g = blockIdx.z;
  float acc[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) acc[v] = 0.f;
  if (c < C) {
    long long r0 = (long long)chunk * rows_per_chunk;
    long long r1 = min(rows_per_group, r0 + rows_per_chunk);
    long long base = (long long)g * rows_per_group;
    for (long long r = r0 + threadIdx.y; r < r1; r += CR_Y) {
      float v[NV];
      f(base + r, c, C, r, v);
#pragma unroll
      for (int k = 0; k < NV; ++k) acc[k] += v[k];
    }
  }
#pragma unroll
  for (int v = 0; v < NV; ++v) sh[v][threadIdx.y][threadIdx.x] = acc[v];
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      float s = 0.f;
#pragma unroll
      for (int y = 0; y < CR_Y; ++y) s += sh[v][y][threadIdx.x];
      partial[(((long long)g * chunks + chunk) * NV + v) * C + c] = s;
    }
  }
  if (!counters) return;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0) s_ticket = atomicAdd(&counters[(size_t)g * gridDim.x + blockIdx.x], 1u);
  __syncthreads();
  if (s_ticket != (unsigned)(chunks - 1)) return;
  __threadfence();
  float* outs[2] = {out0, out1};
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    float s = 0.f;
    if (c < C && outs[v])
      for (int k = threadIdx.y; k < chunks; k += CR_Y) s += __ldcg(&partial[(((long long)g * chunks + k) * NV + v) * C + c]);
    sh[v][threadIdx.y][threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      if (!outs[v]) continue;
      float s = 0.f;
#pragma unroll
      for (int y = 0; y < CR_Y; ++y) s += sh[v][y][threadIdx.x];
      outs[v][(long long)g * C + c] = s * scale;
    }
  }
  if (threadIdx.x == 0 && threadIdx.y == 0) counters[(size_t)g * gridDim.x + blockIdx.x] = 0u;
}

// out_v[g*C + c] = scale * sum_chunk partial.  Block = 32 columns x 8 chunk lanes: the (up to ~150) partials of a column
// are summed by 8 threads in parallel and combined in a fixed order, instead of one long chain of dependent loads.
template <int NV>
__global__ void colreduce_final_kernel(const float* __restrict__ partial, int groups, int chunks, int C, float scale,
                                       float* out0, float* out1) {
  __shared__ float red[NV][8][32];
  const long long i = (long long)blockIdx.x * 32 + threadIdx.x;
  const bool ok = i < (long long)groups * C;
  const int g = ok ? (int)(i / C) : 0, c = ok ? (int)(i % C) : 0;
  float* outs[2] = {out0, out1};
#pragma unroll
  for (int v = 0; v < NV; ++v) {
    float s = 0.f;
    if (ok && outs[v])
      for (int k = threadIdx.y; k < chunks; k += 8) s += partial[(((long long)g * chunks + k) * NV + v) * C + c];
    red[v][threadIdx.y][threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.y == 0 && ok) {
#pragma unroll
    for (int v = 0; v < NV; ++v) {
      if (!outs[v]) continue;
      float s = 0.f;
#pragma unroll
      for (int y = 0; y < 8; ++y) s += red[v][y][threadIdx.x];
      outs[v][i] = s * scale;
    }
  }
}

template <class F, int NV>
int colreduce(cgan_ctx* ctx, F f, int groups, long long rows_per_group, int C, float scale, float* out0, float* out1) {
  int cblocks = cdiv(C, CR_X);
  long long want = (4ll * ctx->num_sms + (long long)cblocks * groups - 1) / ((long long)cblocks * groups);
  long long maxchunks = (rows_per_group + 4 * CR_Y - 1) / (4 * CR_Y);
  long long chunks = want < 1 ? 1 : want;
  if (chunks > maxchunks) chunks = maxchunks;
  if (chunks < 1) chunks = 1;
  if (chunks > 65535) chunks = 65535;
  long long rpc = (rows_per_group + chunks - 1) / chunks;
  rpc = (rpc + CR_Y - 1) / CR_Y * CR_Y;
  chunks = (rows_per_group + rpc - 1) / rpc;
  if (chunks < 1) chunks = 1;
  if (groups > 65535) return cgan_fail(ctx, CGAN_ERR_ARG, "%s: too many groups%s", "colreduce");
  void* ws = nullptr;
  int rc = cgan_ws(ctx, (size_t)groups * chunks * NV * C * sizeof(float), &ws);
  if (rc) return rc;
  float* partial = reinterpret_cast<float*>(ws);
  dim3 grid(cblocks, (unsigned)chunks, groups), block(CR_X, CR_Y);
  if (ctx->counters && (long long)cblocks * groups <= CGAN_NUM_COUNTERS) {     // one launch: the last block per column block finishes
    colreduce_kernel<F, NV><<<grid, block, 0, ctx->stream>>>(f, partial, rows_per_group, C, rpc, (int)chunks, ctx->counters, scale,
                                                             out0, out1);
    CGAN_LAUNCHED(ctx);
    return CGAN_OK;
  }
  colreduce_kernel<F, NV><<<grid, block, 0, ctx->stream>>>(f, partial, rows_per_group, C, rpc, (int)chunks, nullptr, scale, out0, out1);
  CGAN_LAUNCHED(ctx);
  long long tot = (long long)groups * C;
  colreduce_final_kernel<NV><<<cdiv(tot, 32), dim3(32, 8), 0, ctx->stream>>>(partial, groups, (int)chunks, C, scale, out0, out1);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

__global__ void bn_finalize_kernel(float* mean_var, const float* stats, int C, float* mm, float* mv, float decay) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float mean = stats[c], msq = stats[C + c];
  float var = msq - mean * mean;
  mean_var[c] = mean;
  mean_var[C + c] = var;
  if (mm) mm[c] -= (mm[c] - mean) * (1.0f - decay);
  if (mv) mv[c] -= (mv[c] - var) * (1.0f - decay);
}

__global__ void bn_accumulate_kernel(float* mean_var, const float* batch, int C, float* am, float* av, float* ac,
                                     const float* upd) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  bool update = (*upd == 1.0f);
  float counter = *ac + (update ? 1.0f : 0.0f);
  if (c < C) {
    float m = am[c], v = av[c];
    if (update) {
      m += batch[c];
      v += batch[C + c];
      am[c] = m;
      av[c] = v;
    }
    mean_var[c] = m / counter;
    mean_var[C + c] = v / counter;
  }
}

// runs after bn_accumulate_kernel on the same stream: every block of that kernel read the OLD counter
__global__ void bn_accu_counter_kernel(float* ac, const float* upd) {
  if (*upd == 1.0f) *ac += 1.0f;
}

// act: bit 0 = ReLU, CGAN_ACT_ROUND_TF32 = store TF32-rounded values
__global__ void bn_apply_kernel(float* __restrict__ y, const float* __restrict__ x, long long total, int C,
                                long long rows_per_sample, const float* __restrict__ mean_var, float eps,
                                const float* __restrict__ gamma, const float* __restrict__ beta, int cond, int act) {
  const int relu = act & 1, rnd = (act & CGAN_ACT_ROUND_TF32) ? 1 : 0;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    int c = (int)(i % C);
    long long r = i / C;
    long long pidx = cond ? (r / rows_per_sample) * C + c : c;
    float inv = 1.0f / sqrtf(mean_var[C + c] + eps);
    float v = (x[i] - mean_var[c]) * inv;
    if (gamma) v *= gamma[pidx];
    if (beta) v += beta[pidx];
    if (relu) v = fmaxf(v, 0.f);
    y[i] = rnd ? rna_tf32(v) : v;
  }
}

// float4 form (C % 4 == 0, fewer than 2^31 vectors, 16-byte aligned tensors): one 32-bit division per four elements, the
// per-channel parameters come in as float4s from L1
__global__ void bn_apply_v4_kernel(float4* __restrict__ y, const float4* __restrict__ x, unsigned total4, unsigned lanes,
                                   unsigned rows_per_sample, const float* __restrict__ mean_var, float eps,
                                   const float* __restrict__ gamma, const float* __restrict__ beta, int cond, int act) {
  const int relu = act & 1, rnd = (act & CGAN_ACT_ROUND_TF32) ? 1 : 0;
  const unsigned C = lanes * 4;
  const unsigned stride = gridDim.x * blockDim.x;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += stride) {
    const unsigned r = i / lanes, c = (i - r * lanes) * 4;
    const float4 m = *reinterpret_cast<const float4*>(mean_var + c);
    const float4 vv = *reinterpret_cast<const float4*>(mean_var + C + c);
    float4 v = x[i];
    v.x = (v.x - m.x) * (1.0f / sqrtf(vv.x + eps)); v.y = (v.y - m.y) * (1.0f / sqrtf(vv.y + eps));
    v.z = (v.z - m.z) * (1.0f / sqrtf(vv.z + eps)); v.w = (v.w - m.w) * (1.0f / sqrtf(vv.w + eps));
    const size_t pidx = cond ? (size_t)(r / rows_per_sample) * C + c : c;
    if (gamma) { const float4 g = *reinterpret_cast<const float4*>(gamma + pidx); v.x *= g.x; v.y *= g.y; v.z *= g.z; v.w *= g.w; }
    if (beta) { const float4 b = *reinterpret_cast<const float4*>(beta + pidx); v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w; }
    if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    if (rnd) { v.x = rna_tf32(v.x); v.y = rna_tf32(v.y); v.z = rna_tf32(v.z); v.w = rna_tf32(v.w); }
    y[i] = v;
  }
}

// sums[c] = sum_g gamma(g,c)*B(g,c); sums[C+c] = sum_g gamma(g,c)*A(g,c);  A = sum dy*xhat, B = sum dy (per group)
__global__ void bn_bwd_sums_kernel(float* sums, const float* A, const float* Bv, const float* gamma, int groups, int C,
                                   int cond) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s1 = 0.f, s2 = 0.f;
  for (int g = 0; g < groups; ++g) {
    float gm = gamma ? (cond ? gamma[(long long)g * C + c] : gamma[c]) : 1.0f;
    s1 += gm * Bv[(long long)g * C + c];
    s2 += gm * A[(long long)g * C + c];
  }
  sums[c] = s1;
  sums[C + c] = s2;
}

__global__ void bn_bwd_apply_kernel(float* __restrict__ dx, const float* __restrict__ dy, const float* __restrict__ x,
                                    long long total, int C, long long rows_per_sample,
                                    const float* __restrict__ mean_var, float eps, const float* __restrict__ gamma,
                                    int cond, const float* __restrict__ sums, float inv_count, int rnd) {
  long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    int c = (int)(i % C);
    long long r = i / C;
    float inv = 1.0f / sqrtf(mean_var[C + c] + eps);
    float xh = (x[i] - mean_var[c]) * inv;
    float g = gamma ? gamma[cond ? (r / rows_per_sample) * C + c : c] : 1.0f;
    float dxh = dy[i] * g;
    float v = inv * (dxh - sums[c] * inv_count - xh * sums[C + c] * inv_count);
    dx[i] = rnd ? rna_tf32(v) : v;
  }
}

__global__ void bn_bwd_apply_v4_kernel(float4* __restrict__ dx, const float4* __restrict__ dy, const float4* __restrict__ x,
                                       unsigned total4, unsigned lanes, unsigned rows_per_sample,
                                       const float* __restrict__ mean_var, float eps, const float* __restrict__ gamma,
                                       int cond, const float* __restrict__ sums, float inv_count, int rnd) {
  const unsigned C = lanes * 4;
  const unsigned stride = gridDim.x * blockDim.x;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += stride) {
    const unsigned r = i / lanes, c = (i - r * lanes) * 4;
    const float4 m = *reinterpret_cast<const float4*>(mean_var + c);
    const float4 vv = *reinterpret_cast<const float4*>(mean_var + C + c);
    const float4 s1 = *reinterpret_cast<const float4*>(sums + c);
    const float4 s2 = *reinterpret_cast<const float4*>(sums + C + c);
    float4 g = make_float4(1.f, 1.f, 1.f, 1.f);
    if (gamma) g = *reinterpret_cast<const float4*>(gamma + (cond ? (size_t)(r / rows_per_sample) * C + c : c));
    const float4 xv = x[i], gy = dy[i];
    float4 o;
    {
      const float inv = 1.0f / sqrtf(vv.x + eps), xh = (xv.x - m.x) * inv;
      o.x = inv * (gy.x * g.x - s1.x * inv_count - xh * s2.x * inv_count);
    }
    {
      const float inv = 1.0f / sqrtf(vv.y + eps), xh = (xv.y - m.y) * inv;
      o.y = inv * (gy.y * g.y - s1.y * inv_count - xh * s2.y * inv_count);
    }
    {
      const float inv = 1.0f / sqrtf(vv.z + eps), xh = (xv.z - m.z) * inv;
      o.z = inv * (gy.z * g.z - s1.z * inv_count - xh * s2.z * inv_count);
    }
    {
      const float inv = 1.0f / sqrtf(vv.w + eps), xh = (xv.w - m.w) * inv;
      o.w = inv * (gy.w * g.w - s1.w * inv_count - xh * s2.w * inv_count);
    }
    if (rnd) { o.x = rna_tf32(o.x); o.y = rna_tf32(o.y); o.z = rna_tf32(o.z); o.w = rna_tf32(o.w); }
    dx[i] = o;
  }
}

// one warp per row: out[r] = sum_c w[r,c]*b[c]
__global__ void gemv_rows_kernel(float* __restrict__ out, const float* __restrict__ w, const float* __restrict__ b,
                                 int rows, int cols) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const float* row = w + (long long)warp * cols;
  float s = 0.f;
  for (int c = lane; c < cols; c += 32) s += row[c] * b[c];
  s = warp_sum(s);
  if (lane == 0) out[warp] = s;
}

// out = t * rsqrt(max(sum t^2, eps)); optionally sigma = dot(out, t).  Single block.
__global__ void l2_normalize_kernel(float* out, const float* t, int n, float eps, float* sigma) {
  __shared__ float sh[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += t[i] * t[i];
  s = block_sum(s, sh);
  float scale = 1.0f / sqrtf(fmaxf(s, eps));
  float d = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float o = t[i] * scale;
    out[i] = o;
    d += o * t[i];
  }
  if (sigma) {
    d = block_sum(d, sh);
    if (threadIdx.x == 0) *sigma = d;
  }
}

__global__ void sn_bwd_kernel(float* __restrict__ dw, const float* __restrict__ dwbar, int rows, int cols, int left,
                              const float* __restrict__ u, const float* __restrict__ v, const float* sigma,
                              const float* dotp) {
  long long total = (long long)rows * cols;
  long long stride = (long long)gridDim.x * blockDim.x;
  float inv_s = 1.0f / *sigma, dp = *dotp;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    int r = (int)(i / cols), c = (int)(i % cols);
    float outer = left ? u[r] * v[c] : v[r] * u[c];
    dw[i] = (dwbar[i] - dp * outer) * inv_s;
  }
}

// ---- batched spectral norm: ONE launch runs the power iteration of every small weight of a network ----------------
// A discriminator call site of resnet_cifar10 / SNDCGAN touches 8-13 spectrally normalised kernels of at most a few
// hundred KB each; run separately that is ~7 tiny launches per kernel (two GEMVs with their finishing passes, two
// normalisations, the scale, the copy of u) = hundreds of launches per training cycle.  Here one CTA per weight does the
// whole of arch_ops.py:503-531 out of L2: t = W^T u (or W u), v = normalize(t), s = W v (or v W), u' = normalize(s),
// sigma = <u', s>, wbar = W / sigma, u <- u', plus the copy of u' the backward needs.  Fixed summation order.
__device__ __forceinline__ void sn_coldot(float* out, const float* __restrict__ w, const float* x, int rows, int cols, float* red) {
  // out[c] = sum_r w[r, c] * x[r]; thread (c, l): column c of a 32..1024-wide block, row lane l
  for (int cb = 0; cb < cols; cb += 1024) {
    const int cw = min(1024, cols - cb);
    int cpad = 32;
    while (cpad < cw) cpad <<= 1;
    const int lanes = 1024 / cpad;
    const int c = threadIdx.x % cpad, l = threadIdx.x / cpad;
    float acc = 0.f;
    if (c < cw)
      for (int r = l; r < rows; r += lanes) acc = fmaf(w[(size_t)r * cols + cb + c], x[r], acc);
    red[threadIdx.x] = acc;
    __syncthreads();
    if (l == 0 && c < cw) {
      float sum = 0.f;
      for (int j = 0; j < lanes; ++j) sum += red[j * cpad + c];
      out[cb + c] = sum;
    }
    __syncthreads();
  }
}
__device__ __forceinline__ void sn_rowdot(float* out, const float* __restrict__ w, const float* x, int rows, int cols) {
  // out[r] = sum_c w[r, c] * x[c]; one warp per row
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < rows; r += 32) {
    float acc = 0.f;
    for (int c = lane; c < cols; c += 32) acc = fmaf(w[(size_t)r * cols + c], x[c], acc);
    acc = warp_sum(acc);
    if (lane == 0) out[r] = acc;
  }
  __syncthreads();
}
__device__ __forceinline__ float sn_normalize(float* v, int n, float eps, float* sh, float* dot_with_raw) {
  // v <- v * rsqrt(max(sum v^2, eps)); returns via *dot_with_raw the dot product of the normalised and the raw vector
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += v[i] * v[i];
  s = block_sum(s, sh);
  const float scale = 1.0f / sqrtf(fmaxf(s, eps));
  float d = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float raw = v[i], o = raw * scale;
    v[i] = o;
    d += o * raw;
  }
  d = block_sum(d, sh);
  if (dot_with_raw) *dot_with_raw = d;
  return scale;
}

__global__ void __launch_bounds__(1024, 1)
sn_batched_kernel(const cgan_sn_item* __restrict__ items, float eps, float* wbar_base, float* v_base, float* sigma_base,
                  float* u_used_base) {
  extern __shared__ float sn_smem[];
  __shared__ float sh[32];
  const cgan_sn_item it = items[blockIdx.x];
  const int rows = it.rows, cols = it.cols;
  const int nu = it.left ? rows : cols, nv = it.left ? cols : rows;
  float* red = sn_smem;                 // 1024 floats
  float* uv = red + 1024;               // u (nu floats)
  float* vv = uv + nu;                  // v (nv floats)
  for (int i = threadIdx.x; i < nu; i += blockDim.x) uv[i] = it.u[i];
  __syncthreads();
  if (it.left) sn_coldot(vv, it.w, uv, rows, cols, red); else sn_rowdot(vv, it.w, uv, rows, cols);
  sn_normalize(vv, nv, eps, sh, nullptr);
  __syncthreads();
  if (it.left) sn_rowdot(uv, it.w, vv, rows, cols); else sn_coldot(uv, it.w, vv, rows, cols, red);
  float sigma;
  sn_normalize(uv, nu, eps, sh, &sigma);
  __syncthreads();
  float* v_out = v_base + it.v_off;
  float* u_used = u_used_base + it.u_off;
  for (int i = threadIdx.x; i < nv; i += blockDim.x) v_out[i] = vv[i];
  for (int i = threadIdx.x; i < nu; i += blockDim.x) {
    const float un = uv[i];
    it.u[i] = un;
    u_used[i] = un;
  }
  if (threadIdx.x == 0) sigma_base[blockIdx.x] = sigma;
  float* wbar = wbar_base + it.wbar_off;
  const size_t n = (size_t)rows * cols;
  for (size_t i = threadIdx.x; i < n; i += blockDim.x) wbar[i] = it.w[i] / sigma;    // "w / norm_value" (arch_ops.py:531)
}

inline bool v4_ok(const void* a, const void* b, const void* c, const void* d, const void* e, const void* f) {
  return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
           reinterpret_cast<uintptr_t>(d) | reinterpret_cast<uintptr_t>(e) | reinterpret_cast<uintptr_t>(f)) & 15) == 0;
}

// ---- layer norm (arch_ops.py:448-450, tf.contrib.layers.layer_norm with begin_norm_axis=1, begin_params_axis=-1) ----
// Sample i of x is the contiguous span [i*span, (i+1)*span), span = h*w*c; its moments run over the whole span, gamma and
// beta are per channel (c = element index mod C).  stats[2i] = mean, stats[2i+1] = r = rsqrt(var + eps).  The per-sample
// reductions split each span over several CTAs (so that a batch of 64 still fills the GPU), accumulate in float64 and
// merge the CTA partials in chunk order in the last CTA of each sample (ticket counter, reset by that CTA): deterministic,
// one launch, no atomics on values.

constexpr int LN_THREADS = 256;

struct LnMomentsF {      // shifted by the sample's first element, so the float64 second moment does not cancel
  const float* x;
  __device__ __forceinline__ void operator()(int i, long long span, long long j, int, double* v) const {
    const double d = (double)x[i * span + j] - (double)x[i * span];
    v[0] = d;
    v[1] = d * d;
  }
};

struct LnBwdSumsF {      // a = gamma*g: sum a, sum a*xhat
  const float *g, *x, *stats, *gamma;
  __device__ __forceinline__ void operator()(int i, long long span, long long j, int c, double* v) const {
    const float xh = (x[i * span + j] - stats[2 * i]) * stats[2 * i + 1];
    const float a = gamma[c] * g[i * span + j];
    v[0] = a;
    v[1] = (double)a * xh;
  }
};

struct LnBwdBwdSumsF {   // sum a, sum a*xhat, sum w, sum w*xhat, sum w*a
  const float *w, *g, *x, *stats, *gamma;
  __device__ __forceinline__ void operator()(int i, long long span, long long j, int c, double* v) const {
    const long long e = i * span + j;
    const float xh = (x[e] - stats[2 * i]) * stats[2 * i + 1];
    const float a = gamma[c] * g[e], wv = w[e];
    v[0] = a;
    v[1] = (double)a * xh;
    v[2] = wv;
    v[3] = (double)wv * xh;
    v[4] = (double)wv * a;
  }
};

// What ln_sample_reduce_kernel writes per sample: the NV means, or (NV = 2 shifted sums, merged over chunks with Chan et
// al.'s pairwise update) mean and rsqrt(var + eps), or mean and var.
enum LnOut { LN_MEANS, LN_MEAN_RSTD, LN_MEAN_VAR };

// grid (chunks, n).  LN_MEANS: out[i*NV + v] = (sum over the span) / span; otherwise out[2i], out[2i+1] as LnOut says.
template <class F, int NV, LnOut OUT>
__global__ void __launch_bounds__(LN_THREADS) ln_sample_reduce_kernel(F f, long long span, int C, long long per_chunk,
                                                                      double* __restrict__ partial, unsigned* counters,
                                                                      float* out, float eps) {
  __shared__ double sh[LN_THREADS / 32][NV];
  __shared__ unsigned s_ticket;
  const int i = blockIdx.y, k = blockIdx.x, chunks = gridDim.x;
  const long long j0 = (long long)k * per_chunk, j1 = min(span, j0 + per_chunk);
  double acc[NV];
#pragma unroll
  for (int v = 0; v < NV; ++v) acc[v] = 0.0;
  long long j = j0 + threadIdx.x;
  int c = (int)(j % C);
  const int step = LN_THREADS % C;
#pragma unroll 4
  for (; j < j1; j += LN_THREADS) {
    double v[NV];
    f(i, span, j, c, v);
#pragma unroll
    for (int q = 0; q < NV; ++q) acc[q] += v[q];
    c += step;
    if (c >= C) c -= C;
  }
#pragma unroll
  for (int v = 0; v < NV; ++v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[v] += __shfl_xor_sync(0xffffffffu, acc[v], o);
  }
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int v = 0; v < NV; ++v) sh[threadIdx.x >> 5][v] = acc[v];
  __syncthreads();
  if (threadIdx.x < NV) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < LN_THREADS / 32; ++w) s += sh[w][threadIdx.x];
    partial[((long long)i * chunks + k) * NV + threadIdx.x] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_ticket = atomicAdd(&counters[i], 1u);
  __syncthreads();
  if (s_ticket != (unsigned)(chunks - 1)) return;
  __threadfence();
  if (threadIdx.x != 0) return;
  const double* p = partial + (long long)i * chunks * NV;
  if constexpr (OUT != LN_MEANS) {
    double n = 0.0, mean = 0.0, m2 = 0.0;          // of the shifted values
    for (int q = 0; q < chunks; ++q) {
      const double nb = (double)(min(span, (long long)(q + 1) * per_chunk) - (long long)q * per_chunk);
      const double s = __ldcg(p + 2 * q), ss = __ldcg(p + 2 * q + 1);
      const double mb = s / nb, m2b = fmax(ss - s * mb, 0.0);
      const double tot = n + nb, delta = mb - mean;
      mean += delta * nb / tot;
      m2 += m2b + delta * delta * n * nb / tot;
      n = tot;
    }
    out[2 * i] = (float)(mean + (double)f.x[(long long)i * span]);
    out[2 * i + 1] = OUT == LN_MEAN_VAR ? (float)(m2 / n) : (float)(1.0 / sqrt(m2 / n + (double)eps));
  } else {
    for (int v = 0; v < NV; ++v) {
      double s = 0.0;
      for (int q = 0; q < chunks; ++q) s += __ldcg(p + q * NV + v);
      out[(long long)i * NV + v] = (float)(s / (double)span);
    }
  }
  counters[i] = 0u;
}

template <class F, int NV, LnOut OUT>
int ln_sample_reduce(cgan_ctx* ctx, F f, int n, long long span, int C, float* out, float eps) {
  if (!ctx->counters) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: no ticket counters on this context%s", "layer norm");
  long long want = (8ll * ctx->num_sms + n - 1) / n;
  long long maxchunks = (span + 4 * LN_THREADS - 1) / (4 * LN_THREADS);
  long long chunks = want < maxchunks ? want : maxchunks;
  if (chunks < 1) chunks = 1;
  long long per = (span + chunks - 1) / chunks;
  chunks = (span + per - 1) / per;
  void* ws = nullptr;
  int rc = cgan_ws(ctx, (size_t)n * chunks * NV * sizeof(double), &ws);
  if (rc) return rc;
  ln_sample_reduce_kernel<F, NV, OUT><<<dim3((unsigned)chunks, (unsigned)n), LN_THREADS, 0, ctx->stream>>>(
      f, span, C, per, reinterpret_cast<double*>(ws), ctx->counters, out, eps);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

// W consecutive elements (W = 4: float4 loads / stores, needs C % 4 == 0 and 16-byte aligned tensors)
template <int W>
__device__ __forceinline__ void ldw(float* v, const float* p) {
  if (W == 4) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    v[0] = *p;
  }
}
template <int W>
__device__ __forceinline__ void stw(float* p, const float* v) {
  if (W == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  else *p = v[0];
}

// Elementwise passes: grid (blocks per sample, n); thread t of a sample handles elements j = (t + k*stride)*W.
#define LN_EW_LOOP(W)                                                                  \
  const int i = blockIdx.y;                                                            \
  const long long stride = (long long)gridDim.x * blockDim.x * W;                      \
  long long j = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * W;                \
  int c = (int)(j % C);                                                                \
  const int step = (int)(stride % C);                                                  \
  for (; j < span; j += stride, c = (c + step >= C) ? c + step - C : c + step)

template <int W>
__global__ void ln_apply_kernel(float* __restrict__ y, const float* __restrict__ x, long long span, int C,
                                const float* __restrict__ stats, const float* __restrict__ gamma,
                                const float* __restrict__ beta, int act) {
  const int relu = act & 1, rnd = (act & CGAN_ACT_ROUND_TF32) ? 1 : 0;
  LN_EW_LOOP(W) {
    const float mean = stats[2 * i], r = stats[2 * i + 1];
    const long long e = (long long)i * span + j;
    float v[W], gm[W], bt[W];
    ldw<W>(v, x + e);
    ldw<W>(gm, gamma + c);
    ldw<W>(bt, beta + c);
#pragma unroll
    for (int q = 0; q < W; ++q) {
      float o = (v[q] - mean) * (r * gm[q]) + bt[q];
      if (relu) o = fmaxf(o, 0.f);
      v[q] = rnd ? rna_tf32(o) : o;
    }
    stw<W>(y + e, v);
  }
}

// dx = r * (a - mean(a) - xhat * mean(a*xhat)), a = gamma*g; sums[2i] = mean(a), sums[2i+1] = mean(a*xhat)
template <int W>
__global__ void ln_bwd_dx_kernel(float* __restrict__ dx, const float* __restrict__ g, const float* __restrict__ x,
                                 long long span, int C, const float* __restrict__ stats, const float* __restrict__ gamma,
                                 const float* __restrict__ sums, int rnd) {
  LN_EW_LOOP(W) {
    const float mean = stats[2 * i], r = stats[2 * i + 1], abar = sums[2 * i], m = sums[2 * i + 1];
    const long long e = (long long)i * span + j;
    float xv[W], gv[W], gm[W];
    ldw<W>(xv, x + e);
    ldw<W>(gv, g + e);
    ldw<W>(gm, gamma + c);
#pragma unroll
    for (int q = 0; q < W; ++q) {
      const float xh = (xv[q] - mean) * r;
      const float o = r * (gm[q] * gv[q] - abar - xh * m);
      xv[q] = rnd ? rna_tf32(o) : o;
    }
    stw<W>(dx + e, xv);
  }
}

// vjp of (g, x, gamma) -> dx for the cotangent w, with P(w) = w - mean(w) - xhat*mean(w*xhat):
//   d_g = gamma * r * P(w)
//   d_x = -r^2 * (xhat * (A - 3 m q) + q * (a - abar) + m * w),  A = mean(w*a) - abar*wbar, m = mean(a*xhat), q = mean(w*xhat)
// d_x is TF's: the variance of tf.nn.moments reads stop_gradient(mean), which drops the term -r^2 * m * (-wbar) of the
// exact second derivative.  s5[5i..5i+4] = mean(a), mean(a*xhat), mean(w), mean(w*xhat), mean(w*a).
template <int W>
__global__ void ln_bwd_bwd_kernel(float* __restrict__ d_g, float* __restrict__ d_x, const float* __restrict__ w,
                                  const float* __restrict__ g, const float* __restrict__ x, long long span, int C,
                                  const float* __restrict__ stats, const float* __restrict__ gamma,
                                  const float* __restrict__ s5, int rnd) {
  LN_EW_LOOP(W) {
    const float mean = stats[2 * i], r = stats[2 * i + 1];
    const float abar = s5[5 * i], m = s5[5 * i + 1], wbar = s5[5 * i + 2], q = s5[5 * i + 3];
    const float A = s5[5 * i + 4] - abar * wbar, r2 = r * r;
    const long long e = (long long)i * span + j;
    float xv[W], gv[W], wv[W], gm[W], og[W];
    ldw<W>(xv, x + e);
    ldw<W>(gv, g + e);
    ldw<W>(wv, w + e);
    ldw<W>(gm, gamma + c);
#pragma unroll
    for (int k = 0; k < W; ++k) {
      const float xh = (xv[k] - mean) * r, a = gm[k] * gv[k];
      og[k] = gm[k] * r * (wv[k] - wbar - xh * q);
      const float o = -r2 * (xh * (A - 3.f * m * q) + q * (a - abar) + m * wv[k]);
      xv[k] = rnd ? rna_tf32(o) : o;
    }
    if (d_g) stw<W>(d_g + e, og);
    if (d_x) stw<W>(d_x + e, xv);
  }
}
#undef LN_EW_LOOP

// per-channel sums over all pixels (colreduce rows): dgamma = sum g*xhat, dbeta = sum g
struct LnBwdF {
  const float *g, *x, *stats;
  long long hw;
  __device__ __forceinline__ void operator()(long long r, int c, int C, long long, float* v) const {
    const long long i = r / hw;
    const float gv = g[r * C + c];
    v[0] = gv * ((x[r * C + c] - stats[2 * i]) * stats[2 * i + 1]);
    v[1] = gv;
  }
};
// d_gamma of the double backward: sum g * r * P(w)
struct LnBwdBwdGammaF {
  const float *w, *g, *x, *stats, *s5;
  long long hw;
  __device__ __forceinline__ void operator()(long long r, int c, int C, long long, float* v) const {
    const long long i = r / hw;
    const float rr = stats[2 * i + 1], xh = (x[r * C + c] - stats[2 * i]) * rr;
    v[0] = g[r * C + c] * rr * (w[r * C + c] - s5[5 * i + 2] - xh * s5[5 * i + 3]);
  }
};

// grid for the elementwise passes: about 16 blocks per SM in all, at least one per sample
inline dim3 ln_ew_grid(cgan_ctx* ctx, int n, long long span, int w) {
  long long per = ((long long)ctx->num_sms * 16 + n - 1) / n;
  long long need = (span / w + 255) / 256;
  if (per > need) per = need;
  if (per < 1) per = 1;
  return dim3((unsigned)per, (unsigned)n);
}

// per-sample results that must outlive the reduction partials at the head of the workspace (colreduce reuses the head)
int ln_tail(cgan_ctx* ctx, size_t floats, float** out) {
  void* ws = nullptr;
  const size_t need = (floats * sizeof(float) + 255) / 256 * 256;
  int rc = cgan_ws(ctx, need + (size_t)64 * 1024 * 1024, &ws);
  if (rc) return rc;
  *out = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + ctx->ws_bytes - need);
  return CGAN_OK;
}

#define LN_CHECK_SHAPE(ctx, n, span, c)                                                                              \
  CGAN_REQUIRE(ctx, (n) > 0 && (n) <= 65535 && (c) > 0 && (span) > 0 && (span) % (c) == 0,                          \
               "need 0 < n <= 65535 samples and a span that is a positive multiple of the channels")

// ---- DRAGAN perturbation (penalty_lib.py:46-50) ----------------------------------------------------------------------
// clip(x + std * (u - 0.5), 0, 1) with every operation rounded on its own, as TF's graph evaluates it (no FMA)
__device__ __forceinline__ float dragan_noisy(float x, float sd, float u) {
  return fmaxf(fminf(__fadd_rn(x, __fmul_rn(sd, u - 0.5f)), 1.0f), 0.0f);
}

// moments[1] is the batch variance; element i draws u from the stream at offset step * n + i.  n4 > 0: float4 body.
__global__ void dragan_perturb_kernel(float* __restrict__ y, const float* __restrict__ x, long long n, long long n4,
                                      unsigned long long seed, const int32_t* __restrict__ step,
                                      const float* __restrict__ moments, float* __restrict__ std_out) {
  const float sd = __fsqrt_rn(moments[1]);
  if (blockIdx.x == 0 && threadIdx.x == 0) *std_out = sd;
  const unsigned long long off = (unsigned long long)*step * (unsigned long long)n;
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  for (long long v = t0; v < n4; v += stride) {
    const float4 a = reinterpret_cast<const float4*>(x)[v];
    const unsigned long long e = off + 4ull * (unsigned long long)v;
    reinterpret_cast<float4*>(y)[v] = make_float4(
        dragan_noisy(a.x, sd, splitmix_uniform(seed, e)), dragan_noisy(a.y, sd, splitmix_uniform(seed, e + 1)),
        dragan_noisy(a.z, sd, splitmix_uniform(seed, e + 2)), dragan_noisy(a.w, sd, splitmix_uniform(seed, e + 3)));
  }
  for (long long i = 4 * n4 + t0; i < n; i += stride)
    y[i] = dragan_noisy(x[i], sd, splitmix_uniform(seed, off + (unsigned long long)i));
}

// ---- L2 penalty over the kernels of a packed parameter buffer (penalty_lib.py:98-102) --------------------------------
// Segment s = (segs[2s], segs[2s+1]) = (offset, length) in floats.  L2_LANES blocks share a segment, lane l reading the
// float4s l*256 + t, l*256 + t + L2_LANES*256, ...: the summation order depends on this constant and the table only.
constexpr int L2_LANES = 64;
constexpr int L2_THREADS = 256;

__device__ __forceinline__ long long l2_vec4(const float* base, long long off, long long len) {
  return ((reinterpret_cast<uintptr_t>(base + off) & 15) == 0) ? len / 4 : 0;
}

// out[0] = mean over segments of sum(w^2) / 2: float64 squares and sums, per-lane partials merged in lane order and the
// segments in table order by the last block (ticket counter, reset by that block), rounded once to fp32
__global__ void __launch_bounds__(L2_THREADS) l2_penalty_kernel(float* __restrict__ out, const float* __restrict__ p,
                                                                const long long* __restrict__ segs, int nseg,
                                                                double* __restrict__ partial, unsigned* counter) {
  __shared__ double sh[L2_THREADS / 32];
  __shared__ unsigned s_ticket;
  const int s = blockIdx.y, lane = blockIdx.x;
  const long long off = segs[2 * s], len = segs[2 * s + 1], len4 = l2_vec4(p, off, len);
  const float* w = p + off;
  double acc = 0.0;
  for (long long v = (long long)lane * L2_THREADS + threadIdx.x; v < len4; v += (long long)L2_LANES * L2_THREADS) {
    const float4 a = reinterpret_cast<const float4*>(w)[v];
    acc += (double)a.x * a.x;
    acc += (double)a.y * a.y;
    acc += (double)a.z * a.z;
    acc += (double)a.w * a.w;
  }
  for (long long j = 4 * len4 + (long long)lane * L2_THREADS + threadIdx.x; j < len; j += (long long)L2_LANES * L2_THREADS)
    acc += (double)w[j] * w[j];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
    for (int q = 0; q < L2_THREADS / 32; ++q) b += sh[q];
    partial[(long long)s * L2_LANES + lane] = b;
    __threadfence();
    s_ticket = atomicAdd(counter, 1u);
  }
  __syncthreads();
  if (s_ticket != (unsigned)(nseg * L2_LANES - 1)) return;
  __threadfence();
  for (int t = threadIdx.x; t < nseg; t += L2_THREADS) {       // each segment's lanes in order, in place of lane 0
    double ss = 0.0;
    for (int q = 0; q < L2_LANES; ++q) ss += __ldcg(partial + (long long)t * L2_LANES + q);
    partial[(long long)t * L2_LANES] = 0.5 * ss;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double tot = 0.0;
  for (int t = 0; t < nseg; ++t) tot += partial[(long long)t * L2_LANES];
  out[0] = (float)(tot / nseg);
  *counter = 0u;
}

// g[seg] += fp32(fp32(scale[0] * mul) * w[seg]) over the segments only
__global__ void __launch_bounds__(L2_THREADS) l2_penalty_bwd_kernel(float* __restrict__ g, const float* __restrict__ p,
                                                                    const long long* __restrict__ segs,
                                                                    const float* __restrict__ scale, float mul) {
  const int s = blockIdx.y, lane = blockIdx.x;
  const long long off = segs[2 * s], len = segs[2 * s + 1];
  const long long len4 = l2_vec4(p, off, len) > 0 && l2_vec4(g, off, len) > 0 ? len / 4 : 0;
  const float c = __fmul_rn(scale[0], mul);
  const float* w = p + off;
  float* d = g + off;
  for (long long v = (long long)lane * L2_THREADS + threadIdx.x; v < len4; v += (long long)L2_LANES * L2_THREADS) {
    const float4 a = reinterpret_cast<const float4*>(w)[v];
    float4 b = reinterpret_cast<float4*>(d)[v];
    b.x = __fadd_rn(b.x, __fmul_rn(c, a.x));
    b.y = __fadd_rn(b.y, __fmul_rn(c, a.y));
    b.z = __fadd_rn(b.z, __fmul_rn(c, a.z));
    b.w = __fadd_rn(b.w, __fmul_rn(c, a.w));
    reinterpret_cast<float4*>(d)[v] = b;
  }
  for (long long j = 4 * len4 + (long long)lane * L2_THREADS + threadIdx.x; j < len; j += (long long)L2_LANES * L2_THREADS)
    d[j] = __fadd_rn(d[j], __fmul_rn(c, w[j]));
}

}  // namespace

int cgan_colsum(cgan_ctx* ctx, float* out, const float* x, int groups, int64_t rows_per_group, int c) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, out && x && groups > 0 && rows_per_group > 0 && c > 0, "bad argument");
  return colreduce<SumF, 1>(ctx, SumF{x}, groups, rows_per_group, c, 1.0f, out, nullptr);
}

int cgan_bn_moments(cgan_ctx* ctx, float* stats2c, const float* x, int64_t rows, int c) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, stats2c && x && rows > 0 && c > 0, "bad argument");
  return colreduce<MomentsF, 2>(ctx, MomentsF{x}, 1, rows, c, 1.0f / (float)rows, stats2c, stats2c + c);
}

int cgan_bn_finalize(cgan_ctx* ctx, float* mean_var2c, const float* stats2c, int c, float* moving_mean,
                     float* moving_var, float decay) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, mean_var2c && stats2c && c > 0, "bad argument");
  bn_finalize_kernel<<<cdiv(c, 256), 256, 0, ctx->stream>>>(mean_var2c, stats2c, c, moving_mean, moving_var, decay);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_bn_accumulate(cgan_ctx* ctx, float* mean_var2c, const float* batch, int c, float* accu_mean, float* accu_var,
                       float* accu_counter, const float* update_accus_dev) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, mean_var2c && batch && accu_mean && accu_var && accu_counter && update_accus_dev, "null pointer");
  CGAN_REQUIRE(ctx, c > 0, "channels must be positive");
  bn_accumulate_kernel<<<cdiv(c, 256), 256, 0, ctx->stream>>>(mean_var2c, batch, c, accu_mean, accu_var, accu_counter,
                                                              update_accus_dev);
  CGAN_LAUNCHED(ctx);
  bn_accu_counter_kernel<<<1, 1, 0, ctx->stream>>>(accu_counter, update_accus_dev);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_bn_apply(cgan_ctx* ctx, float* y, const float* x, int64_t rows, int c, int64_t rows_per_sample,
                  const float* mean_var2c, float eps, const float* gamma, const float* beta, int cond, int act) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, y && x && mean_var2c && rows > 0 && c > 0, "bad argument");
  CGAN_REQUIRE(ctx, !cond || (rows_per_sample > 0 && rows % rows_per_sample == 0), "rows_per_sample must divide rows");
  CGAN_REQUIRE(ctx, (act & ~(1 | CGAN_ACT_ROUND_TF32)) == 0, "act must be 0 / 1 (ReLU), optionally | CGAN_ACT_ROUND_TF32");
  long long total = (long long)rows * c;
  const long long rps = rows_per_sample > 0 ? rows_per_sample : 1;
  if (c % 4 == 0 && total / 4 < (1ll << 31) && rps < (1ll << 31) && v4_ok(y, x, mean_var2c, gamma, beta, nullptr)) {
    bn_apply_v4_kernel<<<ew_grid(ctx, total / 4), 256, 0, ctx->stream>>>(
        reinterpret_cast<float4*>(y), reinterpret_cast<const float4*>(x), (unsigned)(total / 4), (unsigned)(c / 4), (unsigned)rps,
        mean_var2c, eps, gamma, beta, cond, act);
  } else {
    bn_apply_kernel<<<ew_grid(ctx, total), 256, 0, ctx->stream>>>(y, x, total, c, rps, mean_var2c, eps, gamma, beta, cond, act);
  }
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_bn_bwd_reduce(cgan_ctx* ctx, float* sums2c, float* dgamma, float* dbeta, const float* dy, const float* x,
                       int64_t rows, int c, int64_t rows_per_sample, const float* mean_var2c, float eps,
                       const float* gamma, int cond) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, sums2c && dy && x && mean_var2c && rows > 0 && c > 0, "bad argument");
  CGAN_REQUIRE(ctx, !cond || (rows_per_sample > 0 && rows % rows_per_sample == 0), "rows_per_sample must divide rows");
  int groups = cond ? (int)(rows / rows_per_sample) : 1;
  long long rpg = cond ? rows_per_sample : rows;
  // per-group A = sum dy*xhat, B = sum dy; kept in caller-visible dgamma/dbeta or in workspace tail
  float *A = dgamma, *Bv = dbeta;
  void* ws = nullptr;
  if (!A || !Bv) {
    // scratch behind the colreduce partials: reserve generously first so the pointer stays valid
    size_t need = (size_t)groups * c * 2 * sizeof(float);
    int rc = cgan_ws(ctx, need + (size_t)64 * 1024 * 1024, &ws);
    if (rc) return rc;
    float* tail = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + ctx->ws_bytes - need);
    if (!A) A = tail;
    if (!Bv) Bv = tail + (size_t)groups * c;
  }
  int rc = colreduce<BnBwdF, 2>(ctx, BnBwdF{dy, x, mean_var2c, eps}, groups, rpg, c, 1.0f, A, Bv);
  if (rc) return rc;
  bn_bwd_sums_kernel<<<cdiv(c, 256), 256, 0, ctx->stream>>>(sums2c, A, Bv, gamma, groups, c, cond);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_bn_bwd_apply(cgan_ctx* ctx, float* dx, const float* dy, const float* x, int64_t rows, int c,
                      int64_t rows_per_sample, const float* mean_var2c, float eps, const float* gamma, int cond,
                      const float* sums2c, float inv_count, int round_tf32) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, dx && dy && x && mean_var2c && sums2c && rows > 0 && c > 0, "bad argument");
  long long total = (long long)rows * c;
  const long long rps = rows_per_sample > 0 ? rows_per_sample : 1;
  if (c % 4 == 0 && total / 4 < (1ll << 31) && rps < (1ll << 31) && v4_ok(dx, dy, x, mean_var2c, gamma, sums2c)) {
    bn_bwd_apply_v4_kernel<<<ew_grid(ctx, total / 4), 256, 0, ctx->stream>>>(
        reinterpret_cast<float4*>(dx), reinterpret_cast<const float4*>(dy), reinterpret_cast<const float4*>(x),
        (unsigned)(total / 4), (unsigned)(c / 4), (unsigned)rps, mean_var2c, eps, gamma, cond, sums2c, inv_count, round_tf32 ? 1 : 0);
  } else {
    bn_bwd_apply_kernel<<<ew_grid(ctx, total), 256, 0, ctx->stream>>>(dx, dy, x, total, c, rps, mean_var2c, eps, gamma, cond,
                                                                      sums2c, inv_count, round_tf32 ? 1 : 0);
  }
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_layer_norm_moments(cgan_ctx* ctx, float* stats2n, const float* x, int n, int64_t span, float eps) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, stats2n && x, "null pointer");
  LN_CHECK_SHAPE(ctx, n, span, 1);
  return ln_sample_reduce<LnMomentsF, 2, LN_MEAN_RSTD>(ctx, LnMomentsF{x}, n, span, 1, stats2n, eps);
}

int cgan_layer_norm_apply(cgan_ctx* ctx, float* y, const float* x, int n, int64_t span, int c, const float* stats2n,
                          const float* gamma, const float* beta, int act) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, y && x && stats2n && gamma && beta, "null pointer");
  LN_CHECK_SHAPE(ctx, n, span, c);
  CGAN_REQUIRE(ctx, (act & ~(1 | CGAN_ACT_ROUND_TF32)) == 0, "act must be 0 / 1 (ReLU), optionally | CGAN_ACT_ROUND_TF32");
  if (c % 4 == 0 && v4_ok(y, x, gamma, beta, nullptr, nullptr))
    ln_apply_kernel<4><<<ln_ew_grid(ctx, n, span, 4), 256, 0, ctx->stream>>>(y, x, span, c, stats2n, gamma, beta, act);
  else
    ln_apply_kernel<1><<<ln_ew_grid(ctx, n, span, 1), 256, 0, ctx->stream>>>(y, x, span, c, stats2n, gamma, beta, act);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_layer_norm_bwd(cgan_ctx* ctx, float* dx, float* dgamma, float* dbeta, const float* g, const float* x, int n,
                        int64_t span, int c, const float* stats2n, const float* gamma, int round_tf32) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, g && x && stats2n && gamma, "null pointer");
  LN_CHECK_SHAPE(ctx, n, span, c);
  const long long hw = span / c;
  float* sums = nullptr;
  int rc = ln_tail(ctx, (size_t)2 * n, &sums);
  if (rc) return rc;
  if (dgamma || dbeta) {    // one read of (g, x) for both per-channel sums
    rc = colreduce<LnBwdF, 2>(ctx, LnBwdF{g, x, stats2n, hw}, 1, (long long)n * hw, c, 1.0f, dgamma, dbeta);
    if (rc) return rc;
  }
  if (!dx) return CGAN_OK;
  rc = ln_sample_reduce<LnBwdSumsF, 2, LN_MEANS>(ctx, LnBwdSumsF{g, x, stats2n, gamma}, n, span, c, sums, 0.f);
  if (rc) return rc;
  if (c % 4 == 0 && v4_ok(dx, g, x, gamma, nullptr, nullptr))
    ln_bwd_dx_kernel<4><<<ln_ew_grid(ctx, n, span, 4), 256, 0, ctx->stream>>>(dx, g, x, span, c, stats2n, gamma, sums,
                                                                             round_tf32 ? 1 : 0);
  else
    ln_bwd_dx_kernel<1><<<ln_ew_grid(ctx, n, span, 1), 256, 0, ctx->stream>>>(dx, g, x, span, c, stats2n, gamma, sums,
                                                                             round_tf32 ? 1 : 0);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_layer_norm_bwd_bwd(cgan_ctx* ctx, float* d_g, float* d_x, float* d_gamma, const float* w, const float* g,
                            const float* x, int n, int64_t span, int c, const float* stats2n, const float* gamma,
                            int round_tf32) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, w && g && x && stats2n && gamma, "null pointer");
  LN_CHECK_SHAPE(ctx, n, span, c);
  const long long hw = span / c;
  float* s5 = nullptr;
  int rc = ln_tail(ctx, (size_t)5 * n, &s5);
  if (rc) return rc;
  rc = ln_sample_reduce<LnBwdBwdSumsF, 5, LN_MEANS>(ctx, LnBwdBwdSumsF{w, g, x, stats2n, gamma}, n, span, c, s5, 0.f);
  if (rc) return rc;
  if (d_gamma) {
    rc = colreduce<LnBwdBwdGammaF, 1>(ctx, LnBwdBwdGammaF{w, g, x, stats2n, s5, hw}, 1, (long long)n * hw, c, 1.0f, d_gamma,
                                      nullptr);
    if (rc) return rc;
  }
  if (!d_g && !d_x) return CGAN_OK;
  if (c % 4 == 0 && v4_ok(d_g ? d_g : w, d_x ? d_x : w, w, g, x, gamma))
    ln_bwd_bwd_kernel<4><<<ln_ew_grid(ctx, n, span, 4), 256, 0, ctx->stream>>>(d_g, d_x, w, g, x, span, c, stats2n, gamma, s5,
                                                                              round_tf32 ? 1 : 0);
  else
    ln_bwd_bwd_kernel<1><<<ln_ew_grid(ctx, n, span, 1), 256, 0, ctx->stream>>>(d_g, d_x, w, g, x, span, c, stats2n, gamma, s5,
                                                                              round_tf32 ? 1 : 0);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_dragan_perturb(cgan_ctx* ctx, float* y, const float* x, int64_t n, uint64_t seed, const int32_t* step_dev,
                        float* std_out) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, y && x && step_dev && std_out, "null pointer");
  CGAN_REQUIRE(ctx, n > 0, "need a non-empty batch");
  float* moments = nullptr;
  int rc = ln_tail(ctx, 2, &moments);
  if (rc) return rc;
  // the layer-norm moments of one "sample" spanning the whole batch, its variance instead of rsqrt(var + eps)
  rc = ln_sample_reduce<LnMomentsF, 2, LN_MEAN_VAR>(ctx, LnMomentsF{x}, 1, n, 1, moments, 0.f);
  if (rc) return rc;
  const long long n4 = (al16(x) && al16(y)) ? n / 4 : 0;
  dragan_perturb_kernel<<<ew_grid(ctx, n4 > 0 ? n4 : n), 256, 0, ctx->stream>>>(y, x, n, n4, seed, step_dev, moments,
                                                                                std_out);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_l2_penalty(cgan_ctx* ctx, float* out, const float* flat_param, const int64_t* segs_dev, int nseg) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, out && flat_param && segs_dev, "null pointer");
  CGAN_REQUIRE(ctx, nseg > 0 && nseg <= 65535, "need 0 < nseg <= 65535 segments");
  if (!ctx->counters) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: no ticket counters on this context%s", "l2 penalty");
  void* ws = nullptr;
  int rc = cgan_ws(ctx, (size_t)nseg * L2_LANES * sizeof(double), &ws);
  if (rc) return rc;
  l2_penalty_kernel<<<dim3(L2_LANES, (unsigned)nseg), L2_THREADS, 0, ctx->stream>>>(
      out, flat_param, reinterpret_cast<const long long*>(segs_dev), nseg, reinterpret_cast<double*>(ws), ctx->counters);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_l2_penalty_bwd(cgan_ctx* ctx, float* flat_grad, const float* flat_param, const int64_t* segs_dev, int nseg,
                        const float* scale_dev, float mul) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, flat_grad && flat_param && segs_dev && scale_dev, "null pointer");
  CGAN_REQUIRE(ctx, nseg > 0 && nseg <= 65535, "need 0 < nseg <= 65535 segments");
  l2_penalty_bwd_kernel<<<dim3(L2_LANES, (unsigned)nseg), L2_THREADS, 0, ctx->stream>>>(
      flat_grad, flat_param, reinterpret_cast<const long long*>(segs_dev), scale_dev, mul);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

// internal: out[c] = sum_r w[r,c]*a[r]
static int gemv_cols(cgan_ctx* ctx, float* out, const float* w, const float* a, int rows, int cols) {
  return colreduce<WeightedSumF, 1>(ctx, WeightedSumF{w, a}, 1, rows, cols, 1.0f, out, nullptr);
}
static int gemv_rows(cgan_ctx* ctx, float* out, const float* w, const float* b, int rows, int cols) {
  gemv_rows_kernel<<<cdiv((long long)rows * 32, 256), 256, 0, ctx->stream>>>(out, w, b, rows, cols);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_spectral_norm(cgan_ctx* ctx, const float* w, int rows, int cols, int left, float eps, float* u, float* v,
                       float* sigma, float* wbar) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, w && u && v && sigma && rows > 0 && cols > 0, "bad argument");
  // scratch vector t (max(rows, cols)) lives in the workspace tail, clear of the colreduce partials
  size_t tbytes = (size_t)(rows > cols ? rows : cols) * sizeof(float);
  void* ws = nullptr;
  int rc = cgan_ws(ctx, tbytes + (size_t)64 * 1024 * 1024, &ws);
  if (rc) return rc;
  float* t = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + ctx->ws_bytes - ((tbytes + 255) / 256) * 256);
  if (left) {
    // v = normalize(W^T u); u' = normalize(W v); sigma = u'^T W v       (arch_ops.py:505-509, 525)
    rc = gemv_cols(ctx, t, w, u, rows, cols);
    if (rc) return rc;
    l2_normalize_kernel<<<1, 1024, 0, ctx->stream>>>(v, t, cols, eps, nullptr);
    CGAN_LAUNCHED(ctx);
    rc = gemv_rows(ctx, t, w, v, rows, cols);
    if (rc) return rc;
    l2_normalize_kernel<<<1, 1024, 0, ctx->stream>>>(u, t, rows, eps, sigma);
    CGAN_LAUNCHED(ctx);
  } else {
    // v = normalize(u W^T); u' = normalize(v W); sigma = v W u'^T       (arch_ops.py:511-513, 527)
    rc = gemv_rows(ctx, t, w, u, rows, cols);
    if (rc) return rc;
    l2_normalize_kernel<<<1, 1024, 0, ctx->stream>>>(v, t, rows, eps, nullptr);
    CGAN_LAUNCHED(ctx);
    rc = gemv_cols(ctx, t, w, v, rows, cols);
    if (rc) return rc;
    l2_normalize_kernel<<<1, 1024, 0, ctx->stream>>>(u, t, cols, eps, sigma);
    CGAN_LAUNCHED(ctx);
  }
  if (wbar) return cgan_scale_by_dev(ctx, wbar, w, sigma, 1.0f, 1, (int64_t)rows * cols);
  return CGAN_OK;
}

int cgan_spectral_norm_batched(cgan_ctx* ctx, const cgan_sn_item* items_dev, int n, int max_rows_plus_cols, float eps,
                               float* wbar_base, float* v_base, float* sigma_base, float* u_used_base) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, items_dev && n > 0 && wbar_base && v_base && sigma_base && u_used_base, "bad argument");
  const size_t smem = (size_t)(1024 + max_rows_plus_cols) * sizeof(float);
  CGAN_REQUIRE(ctx, smem <= 200 * 1024, "rows + cols too large for the batched kernel (use cgan_spectral_norm)");
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    CGAN_CUDA(ctx, cudaFuncSetAttribute(sn_batched_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  sn_batched_kernel<<<n, 1024, smem, ctx->stream>>>(items_dev, eps, wbar_base, v_base, sigma_base, u_used_base);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_spectral_norm_bwd(cgan_ctx* ctx, float* dw, const float* dwbar, const float* wbar, int rows, int cols,
                           int left, const float* u, const float* v, const float* sigma) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, dw && dwbar && wbar && u && v && sigma && rows > 0 && cols > 0, "bad argument");
  void* ws = nullptr;
  int rc = cgan_ws(ctx, (size_t)64 * 1024 * 1024, &ws);
  if (rc) return rc;
  float* dotp = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + ctx->ws_bytes - 256);
  rc = cgan_dot(ctx, dotp, dwbar, wbar, (int64_t)rows * cols);
  if (rc) return rc;
  long long total = (long long)rows * cols;
  sn_bwd_kernel<<<ew_grid(ctx, total), 256, 0, ctx->stream>>>(dw, dwbar, rows, cols, left, u, v, sigma, dotp);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}
