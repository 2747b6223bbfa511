// Self-modulated batch norm (arch_ops.py:370-420; Chen et al., "On Self Modulation for GANs"): the per-layer MLP on z
//   h = relu(z W_h + b_h)   [N, H]   (h = z when H = 0)
//   gamma = h W_gamma + b_gamma,  beta = h W_beta + b_beta   [N, C]
// with gamma and beta stored as one [2N, C] buffer `gb` (rows 0..N-1 gamma, N..2N-1 beta), each half in the
// [samples, C] layout cgan_bn_apply(cond = 1) reads.  K = H (or Z when H = 0) is the inner dimension of the wide layer.
//
// Exact fp32 in both math modes, no floating-point atomics: every output is one fmaf chain in a fixed order (over k,
// then + bias; over samples for the weight gradients), and the cross-CTA sum of the hidden gradient is a second launch
// that adds the per-CTA partials in CTA order.  Results do not depend on the stream's history, reruns are bit-identical.
//
// sm_fwd_kernel (forward and tangent): grid (column tiles of the virtual [gamma | beta] column space, row chunks).  A CTA
// computes h for its 64-row chunk into shared memory once, then streams the [K, 128] weight tiles it owns through shared
// memory in 32-row stages and writes 64 x 128 outputs per tile (8 x 4 per thread).  The grid is capped at two CTAs per SM,
// so each CTA owns several tiles and the recomputation of h is amortised; the weights are read once per row chunk.
//
// sm_bwd_kernel: one CTA per SM, each owning a group of 128-column tiles (both halves).  Per 64-sample chunk and tile it stages dgamma and
// dbeta [64, 128], forms dW = h^T dgamma (accumulated over the chunks in sample order, the running sum living in the
// destination) and db, and adds dgamma W_gamma^T + dbeta W_beta^T over its columns into a [64, K] register tile, written
// as this CTA's partial of dh.  sm_bwd_hidden_kernel then adds the partials in CTA order: blocks [0, N) own one sample
// (dh row -> ReLU mask -> dz = dh W_h^T), blocks [N, N + H) one hidden unit (dh column -> mask -> db_h, dW_h = z^T dh).
#include "common.cuh"

namespace {

constexpr int SM_THREADS = 256;
constexpr int SM_ROWS = 64;        // rows (samples / tangent rows) per chunk
constexpr int SM_COLS = 128;       // output columns per tile
constexpr int SM_KC = 32;          // inner-dimension stage of the forward weight tile / column stage of the dh product
constexpr int SM_MAX_K = 256;
constexpr long long SM_PART_BYTES = 64ll << 20;

static_assert(SM_THREADS == 256 && SM_ROWS == 64 && SM_COLS == 128, "thread tile: 8 row groups x 32 column groups");

__device__ __forceinline__ void fma4(float (&acc)[4], float a, float4 b) {
  acc[0] = fmaf(a, b.x, acc[0]);
  acc[1] = fmaf(a, b.y, acc[1]);
  acc[2] = fmaf(a, b.z, acc[2]);
  acc[3] = fmaf(a, b.w, acc[3]);
}

// hs[r][j] (r < 64, row stride K) for rows r0 .. r0 + nr of the hidden layer.  Forward: relu(z W_h + b_h).  Tangent
// (mask != null): (t_z W_h) * [mask[(r0 + r) / kt] > 0].  H = 0: the input rows themselves.  Rows past nr are zero.
__device__ void hidden_rows(float* hs, float* h_out, const float* __restrict__ z, int r0, int nr, int Z, int H,
                            const float* __restrict__ wh, const float* __restrict__ bh, const float* __restrict__ mask,
                            int kt) {
  const int tid = threadIdx.x;
  if (H == 0) {
    for (int e = tid; e < SM_ROWS * Z; e += SM_THREADS) {
      const int r = e / Z;
      hs[e] = r < nr ? z[(long long)(r0 + r) * Z + e % Z] : 0.f;
    }
    return;
  }
  constexpr int PER = 8;
  for (int e0 = 0; e0 < SM_ROWS * H; e0 += SM_THREADS * PER) {
    float acc[PER];
    int rr[PER], jj[PER];
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int e = e0 + i * SM_THREADS + tid;
      rr[i] = e / H;
      jj[i] = e % H;
      acc[i] = 0.f;
    }
    for (int q = 0; q < Z; ++q) {
#pragma unroll
      for (int i = 0; i < PER; ++i)
        if (rr[i] < nr) acc[i] = fmaf(__ldg(z + (long long)(r0 + rr[i]) * Z + q), __ldg(wh + (long long)q * H + jj[i]), acc[i]);
    }
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      if (rr[i] >= SM_ROWS) continue;
      float v = 0.f;
      if (rr[i] < nr) {
        if (mask) {
          v = mask[(long long)((r0 + rr[i]) / kt) * H + jj[i]] > 0.f ? acc[i] : 0.f;
        } else {
          v = acc[i] + bh[jj[i]];
          v = v > 0.f ? v : 0.f;
          if (h_out) h_out[(long long)(r0 + rr[i]) * H + jj[i]] = v;
        }
      }
      hs[rr[i] * H + jj[i]] = v;
    }
  }
}

// out[half * R + r, c] = sum_k hid[r, k] W_half[k, c] (+ b_half[c]) for half 0 (gamma) and 1 (beta)
__global__ void __launch_bounds__(SM_THREADS) sm_fwd_kernel(float* __restrict__ out, float* __restrict__ h_out,
    const float* __restrict__ z, int R, int Z, int H, const float* __restrict__ wh, const float* __restrict__ bh,
    const float* __restrict__ mask, int kt, const float* __restrict__ wg, const float* __restrict__ bg,
    const float* __restrict__ wb, const float* __restrict__ bb, int C, bool vec) {
  extern __shared__ float4 smem4[];
  float* smem = reinterpret_cast<float*>(smem4);
  const int K = H > 0 ? H : Z;
  float* ws = smem;                               // [SM_KC][SM_COLS]
  float* hs = smem + SM_KC * SM_COLS;             // [SM_ROWS][K]
  const int tid = threadIdx.x, tr = tid >> 5, tc = tid & 31;
  const int tiles_c = (C + SM_COLS - 1) / SM_COLS, ntiles = 2 * tiles_c, nchunks = (R + SM_ROWS - 1) / SM_ROWS;
  for (int chunk = blockIdx.y; chunk < nchunks; chunk += gridDim.y) {
    const int r0 = chunk * SM_ROWS, nr = min(SM_ROWS, R - r0);
    __syncthreads();
    hidden_rows(hs, blockIdx.x == 0 ? h_out : nullptr, z, r0, nr, Z, H, wh, bh, mask, kt);
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const int half = t / tiles_c, c0 = (t % tiles_c) * SM_COLS;
      const float* __restrict__ W = half ? wb : wg;
      const float* __restrict__ B = half ? bb : bg;
      float acc[8][4];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
      for (int k0 = 0; k0 < K; k0 += SM_KC) {
        const int kn = min(SM_KC, K - k0);
        __syncthreads();
        if (vec) {
          for (int e = tid; e < SM_KC * SM_COLS / 4; e += SM_THREADS) {
            const int kk = e / (SM_COLS / 4), c = c0 + (e % (SM_COLS / 4)) * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (kk < kn && c < C) v = __ldg(reinterpret_cast<const float4*>(W + (long long)(k0 + kk) * C + c));
            reinterpret_cast<float4*>(ws)[e] = v;
          }
        } else {
          for (int e = tid; e < SM_KC * SM_COLS; e += SM_THREADS) {
            const int kk = e / SM_COLS, c = c0 + e % SM_COLS;
            ws[e] = (kk < kn && c < C) ? __ldg(W + (long long)(k0 + kk) * C + c) : 0.f;
          }
        }
        __syncthreads();
        for (int kk = 0; kk < kn; ++kk) {
          const float4 w = reinterpret_cast<const float4*>(ws + kk * SM_COLS)[tc];
#pragma unroll
          for (int i = 0; i < 8; ++i) fma4(acc[i], hs[(tr * 8 + i) * K + k0 + kk], w);
        }
      }
      const int c = c0 + tc * 4;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = tr * 8 + i;
        if (r >= nr) continue;
        float* o = out + ((long long)half * R + r0 + r) * C + c;
        float v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = (B && c + q < C) ? acc[i][q] + B[c + q] : acc[i][q];
        if (vec && c < C) {
          *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (c + q < C) o[q] = v[q];
        }
      }
    }
  }
}

// shared memory of sm_bwd_kernel: hT [K64][64], dg [2][64][128], wt [SM_KC][KP]
__host__ __device__ __forceinline__ int bwd_k64(int K) { return (K + 63) / 64 * 64; }
__host__ __device__ __forceinline__ int bwd_kp(int K) { return (K + 127) / 128 * 128 + 4; }

template <int NCB>   // column blocks of 128 in the [64, K] dh tile: K <= 128 * NCB
__global__ void __launch_bounds__(SM_THREADS) sm_bwd_kernel(float* __restrict__ dwg, float* __restrict__ dbg,
    float* __restrict__ dwb, float* __restrict__ dbb, float* __restrict__ part, const float* __restrict__ dgb,
    const float* __restrict__ hid, const float* __restrict__ wg, const float* __restrict__ wb, int N, int K, int C,
    bool vec) {
  extern __shared__ float4 smem4[];
  float* smem = reinterpret_cast<float*>(smem4);
  const int K64 = bwd_k64(K), KP = bwd_kp(K);
  float* hT = smem;                                  // [K64][SM_ROWS]
  float* dg = hT + K64 * SM_ROWS;                    // [2][SM_ROWS][SM_COLS]
  float* wt = dg + 2 * SM_ROWS * SM_COLS;            // [SM_KC][KP]
  const int tid = threadIdx.x, tr = tid >> 5, tc = tid & 31;
  const int tiles_c = (C + SM_COLS - 1) / SM_COLS;
  for (int n0 = 0; n0 < N; n0 += SM_ROWS) {
    const int nr = min(SM_ROWS, N - n0);
    float dh[NCB][8][4];
#pragma unroll
    for (int b = 0; b < NCB; ++b)
#pragma unroll
      for (int i = 0; i < 8; ++i) dh[b][i][0] = dh[b][i][1] = dh[b][i][2] = dh[b][i][3] = 0.f;
    __syncthreads();
    for (int e = tid; e < K64 * SM_ROWS; e += SM_THREADS) {
      const int n = e % SM_ROWS, k = e / SM_ROWS;
      hT[e] = (n < nr && k < K) ? hid[(long long)(n0 + n) * K + k] : 0.f;
    }
    for (int t = blockIdx.x; t < tiles_c; t += gridDim.x) {
      const int c0 = t * SM_COLS;
      __syncthreads();
      for (int e = tid; e < 2 * SM_ROWS * SM_COLS; e += SM_THREADS) {
        const int half = e / (SM_ROWS * SM_COLS), n = (e / SM_COLS) % SM_ROWS, c = c0 + e % SM_COLS;
        dg[e] = (n < nr && c < C) ? __ldg(dgb + ((long long)half * N + n0 + n) * C + c) : 0.f;
      }
      __syncthreads();
      const int c = c0 + tc * 4;
      for (int half = 0; half < 2; ++half) {
        float* dw = half ? dwb : dwg;
        float* db = half ? dbb : dbg;
        const float* g = dg + half * SM_ROWS * SM_COLS;
        // dW[k, c] over samples in order, continuing the sum of the previous chunks
        for (int kb = 0; dw && kb < K; kb += SM_ROWS) {
          float acc[8][4];
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int k = kb + tr * 8 + i;
#pragma unroll
            for (int q = 0; q < 4; ++q)
              acc[i][q] = (n0 > 0 && k < K && c + q < C) ? dw[(long long)k * C + c + q] : 0.f;
          }
          for (int n = 0; n < nr; ++n) {
            const float4 b = reinterpret_cast<const float4*>(g + n * SM_COLS)[tc];
#pragma unroll
            for (int i = 0; i < 8; ++i) fma4(acc[i], hT[(kb + tr * 8 + i) * SM_ROWS + n], b);
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const int k = kb + tr * 8 + i;
            if (k >= K) continue;
            float* o = dw + (long long)k * C + c;
            if (vec && c < C) {
              *reinterpret_cast<float4*>(o) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
            } else {
#pragma unroll
              for (int q = 0; q < 4; ++q)
                if (c + q < C) o[q] = acc[i][q];
            }
          }
        }
        if (db && tid < SM_COLS && c0 + tid < C) {
          float s = n0 > 0 ? db[c0 + tid] : 0.f;
          for (int n = 0; n < nr; ++n) s += g[n * SM_COLS + tid];
          db[c0 + tid] = s;
        }
        // dh[n, k] += sum over this tile's columns of g[n, c] W[k, c]
        if (part) {
          const float* __restrict__ W = half ? wb : wg;
          for (int s0 = 0; s0 < SM_COLS; s0 += SM_KC) {
            __syncthreads();
            for (int e = tid; e < SM_KC * K; e += SM_THREADS) {
              const int k = e / SM_KC, cc = e % SM_KC, col = c0 + s0 + cc;
              wt[cc * KP + k] = col < C ? __ldg(W + (long long)k * C + col) : 0.f;
            }
            __syncthreads();
            for (int cc = 0; cc < SM_KC; ++cc) {
#pragma unroll
              for (int b = 0; b < NCB; ++b) {
                const float4 w = reinterpret_cast<const float4*>(wt + cc * KP + b * SM_COLS)[tc];
#pragma unroll
                for (int i = 0; i < 8; ++i) fma4(dh[b][i], g[(tr * 8 + i) * SM_COLS + s0 + cc], w);
              }
            }
          }
        }
      }
    }
    if (part) {
#pragma unroll
      for (int b = 0; b < NCB; ++b)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int n = tr * 8 + i;
          if (n >= nr) continue;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int k = b * SM_COLS + tc * 4 + q;
            if (k < K) part[((long long)blockIdx.x * N + n0 + n) * K + k] = dh[b][i][q];
          }
        }
    }
  }
}

// dh[n, k] = sum over g < G of part[g, n, k] (in g order), times [h[n, k] > 0] when H > 0
__device__ __forceinline__ float dh_value(const float* __restrict__ part, const float* __restrict__ h, int G, int N, int K,
                                          int H, int n, int k) {
  float s = part[(long long)n * K + k];
  for (int g = 1; g < G; ++g) s += part[((long long)g * N + n) * K + k];
  return (H == 0 || h[(long long)n * H + k] > 0.f) ? s : 0.f;
}

__global__ void __launch_bounds__(SM_THREADS) sm_bwd_hidden_kernel(float* __restrict__ dwh, float* __restrict__ dbh,
    float* __restrict__ dz, const float* __restrict__ part, int G, const float* __restrict__ h,
    const float* __restrict__ z, const float* __restrict__ wh, int N, int Z, int H) {
  extern __shared__ float4 smem4[];
  float* s = reinterpret_cast<float*>(smem4);
  const int K = H > 0 ? H : Z;
  const int tid = threadIdx.x;
  if (blockIdx.x < N) {                              // one sample: dz
    if (!dz) return;
    const int n = blockIdx.x;
    for (int k = tid; k < K; k += SM_THREADS) s[k] = dh_value(part, h, G, N, K, H, n, k);
    __syncthreads();
    for (int q = tid; q < Z; q += SM_THREADS) {
      float v;
      if (H == 0) {
        v = s[q];
      } else {
        v = 0.f;
        for (int j = 0; j < H; ++j) v = fmaf(s[j], wh[(long long)q * H + j], v);
      }
      dz[(long long)n * Z + q] = v;
    }
    return;
  }
  const int j = blockIdx.x - N;                      // one hidden unit: db_h, dW_h
  for (int n = tid; n < N; n += SM_THREADS) s[n] = dh_value(part, h, G, N, K, H, n, j);
  __syncthreads();
  if (dbh && tid == 0) {
    float v = 0.f;
    for (int n = 0; n < N; ++n) v += s[n];
    dbh[j] = v;
  }
  if (dwh)
    for (int q = tid; q < Z; q += SM_THREADS) {
      float v = 0.f;
      for (int n = 0; n < N; ++n) v = fmaf(z[(long long)n * Z + q], s[n], v);
      dwh[(long long)q * H + j] = v;
    }
}

int fwd_launch(cgan_ctx* ctx, float* out, float* h_out, const float* z, int R, int Z, int H, const float* wh,
               const float* bh, const float* mask, int kt, const float* wg, const float* bg, const float* wb,
               const float* bb, int C) {
  const int K = H > 0 ? H : Z;
  const size_t smem = (size_t)(SM_KC * SM_COLS + SM_ROWS * K) * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    CGAN_CUDA(ctx, cudaFuncSetAttribute(sm_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (SM_KC * SM_COLS + SM_ROWS * SM_MAX_K) * (int)sizeof(float)));
    attr_set = true;
  }
  const int ntiles = 2 * cdiv(C, SM_COLS), nchunks = cdiv(R, SM_ROWS);
  const int cap = 2 * ctx->num_sms;
  const int gx = ntiles < cap ? ntiles : cap;
  int gy = cap / gx;
  gy = gy < 1 ? 1 : (gy > nchunks ? nchunks : (gy > 65535 ? 65535 : gy));
  const bool vec = (C & 3) == 0 && al16(out) && al16(wg) && al16(wb);
  sm_fwd_kernel<<<dim3(gx, gy), SM_THREADS, smem, ctx->stream>>>(out, h_out, z, R, Z, H, wh, bh, mask, kt, wg, bg, wb, bb, C,
                                                                 vec);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int check_shape(cgan_ctx* ctx, int n, int z_dim, int hidden, int c) {
  CGAN_REQUIRE(ctx, n >= 1 && z_dim >= 1 && hidden >= 0 && c >= 1, "n, z_dim, c >= 1 and hidden >= 0");
  CGAN_REQUIRE(ctx, (hidden > 0 ? hidden : z_dim) <= SM_MAX_K, "the modulation layer's input width (hidden, or z_dim "
               "when hidden = 0) must be <= 256");
  CGAN_REQUIRE(ctx, n <= 12288 && z_dim <= 65536, "n <= 12288 and z_dim <= 65536");
  return CGAN_OK;
}

}  // namespace

int cgan_self_modulation_fwd(cgan_ctx* ctx, float* gb, float* h, const float* z, int n, int z_dim, int hidden,
                             const float* w_h, const float* b_h, const float* w_gamma, const float* b_gamma,
                             const float* w_beta, const float* b_beta, int c) {
  if (!ctx) return CGAN_ERR_ARG;
  if (int rc = check_shape(ctx, n, z_dim, hidden, c)) return rc;
  CGAN_REQUIRE(ctx, gb && z && w_gamma && b_gamma && w_beta && b_beta, "null pointer");
  CGAN_REQUIRE(ctx, hidden == 0 || (h && w_h && b_h), "hidden > 0 needs h, w_h and b_h");
  return fwd_launch(ctx, gb, hidden > 0 ? h : nullptr, z, n, z_dim, hidden, w_h, b_h, nullptr, 1, w_gamma, b_gamma,
                    w_beta, b_beta, c);
}

int cgan_self_modulation_jvp(cgan_ctx* ctx, float* t_gb, const float* t_z, const float* h, const float* w_h,
                             const float* w_gamma, const float* w_beta, int n, int z_dim, int hidden, int c, int k) {
  if (!ctx) return CGAN_ERR_ARG;
  if (int rc = check_shape(ctx, n, z_dim, hidden, c)) return rc;
  CGAN_REQUIRE(ctx, k >= 1 && (long long)n * k < (1ll << 31), "k >= 1 and n * k < 2^31");
  CGAN_REQUIRE(ctx, t_gb && t_z && w_gamma && w_beta, "null pointer");
  CGAN_REQUIRE(ctx, hidden == 0 || (h && w_h), "hidden > 0 needs h and w_h");
  return fwd_launch(ctx, t_gb, nullptr, t_z, n * k, z_dim, hidden, w_h, nullptr, hidden > 0 ? h : nullptr, k, w_gamma,
                    nullptr, w_beta, nullptr, c);
}

int cgan_self_modulation_bwd(cgan_ctx* ctx, float* dw_h, float* db_h, float* dw_gamma, float* db_gamma, float* dw_beta,
                             float* db_beta, float* dz, const float* dgb, const float* h, const float* z,
                             const float* w_h, const float* w_gamma, const float* w_beta, int n, int z_dim, int hidden,
                             int c) {
  if (!ctx) return CGAN_ERR_ARG;
  if (int rc = check_shape(ctx, n, z_dim, hidden, c)) return rc;
  CGAN_REQUIRE(ctx, dgb && z && w_gamma && w_beta, "null pointer");
  CGAN_REQUIRE(ctx, hidden == 0 || (h && w_h), "hidden > 0 needs h and w_h");
  CGAN_REQUIRE(ctx, hidden > 0 || (!dw_h && !db_h), "dw_h / db_h need hidden > 0");
  const int K = hidden > 0 ? hidden : z_dim;
  const bool need_dh = dz || dw_h || db_h;
  const int tiles_c = cdiv(c, SM_COLS);
  int grid = tiles_c < ctx->num_sms ? tiles_c : ctx->num_sms;    // ~180 registers a thread: one CTA per SM
  float* part = nullptr;
  if (need_dh) {
    const long long per_cta = (long long)n * K * (long long)sizeof(float);
    long long cap = SM_PART_BYTES / per_cta;
    if (cap < 1) cap = 1;
    if (grid > cap) grid = (int)cap;
    void* ws = nullptr;
    if (int rc = cgan_ws(ctx, (size_t)(grid * per_cta), &ws)) return rc;
    part = static_cast<float*>(ws);
  }
  const float* hid = hidden > 0 ? h : z;
  const size_t smem = (size_t)(bwd_k64(K) * SM_ROWS + 2 * SM_ROWS * SM_COLS + SM_KC * bwd_kp(K)) * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    const int most = (bwd_k64(SM_MAX_K) * SM_ROWS + 2 * SM_ROWS * SM_COLS + SM_KC * bwd_kp(SM_MAX_K)) * (int)sizeof(float);
    CGAN_CUDA(ctx, cudaFuncSetAttribute(sm_bwd_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
    CGAN_CUDA(ctx, cudaFuncSetAttribute(sm_bwd_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
    attr_set = true;
  }
  const bool vec = (c & 3) == 0 && (!dw_gamma || al16(dw_gamma)) && (!dw_beta || al16(dw_beta));
  if (K <= SM_COLS)
    sm_bwd_kernel<1><<<grid, SM_THREADS, smem, ctx->stream>>>(dw_gamma, db_gamma, dw_beta, db_beta, part, dgb, hid,
                                                             w_gamma, w_beta, n, K, c, vec);
  else
    sm_bwd_kernel<2><<<grid, SM_THREADS, smem, ctx->stream>>>(dw_gamma, db_gamma, dw_beta, db_beta, part, dgb, hid,
                                                             w_gamma, w_beta, n, K, c, vec);
  CGAN_LAUNCHED(ctx);
  if (!need_dh) return CGAN_OK;
  // blocks [0, n): one sample each (they exit at once without dz); [n, n + hidden): one hidden unit each
  const int blocks = n + ((dw_h || db_h) ? hidden : 0);
  const int s_floats = K > n ? K : n;
  sm_bwd_hidden_kernel<<<blocks, SM_THREADS, s_floats * sizeof(float), ctx->stream>>>(dw_h, db_h, dz, part, grid, h, z,
                                                                                    w_h, n, z_dim, hidden);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}
