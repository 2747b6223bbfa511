// k-means of the PRD histograms (metrics/prd_score.py:94-122): k-means++ seeding, Lloyd iterations and the final
// assignment of `groups` independent clusterings of the same points, in float64 throughout.
//
// The hot kernel is km_dist_kernel: x.c for a 128-point x 64-centre tile on the FP64 tensor cores
// (mma.sync m8n8k4 f64), x converted from fp32 when it is staged into shared memory (exact), d and the points padded with
// zeros to the tile.  Its epilogue forms ||x||^2 + ||c||^2 - 2 x.c and finishes the per-group argmin: the 64 columns of a
// CTA hold floor(64 / kk) whole groups of kk centres.  Every output element is the same k-ordered DMMA chain wherever
// its column sits, so a group's distances do not depend on the other groups of the call.
//
// Sums that feed results are taken in a fixed order that does not depend on the launch configuration: the k-means++
// prefix sum is sequential in point order, the centroid sums run over the points in order per (group, cluster, column),
// norms and inertia use fixed per-thread strides and a fixed tree.  Only integer atomics are used (cluster counts).
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace {

constexpr int KM_BM = 128, KM_BN = 64, KM_BK = 32, KM_THREADS = 256;
constexpr int KM_LDS = KM_BK + 4;       // smem row stride (doubles): the fragment loads of a half-warp hit 16 distinct slots
constexpr int KM_LDD = KM_BN + 1;       // epilogue distance tile row stride
constexpr int KM_UPD_COLS = 128;        // columns per CTA of the centroid update
constexpr int KM_MAX_K = 64;

constexpr size_t km_dist_smem() {
  return sizeof(double) * ((size_t)KM_BM * KM_LDD > (size_t)(KM_BM + KM_BN) * KM_LDS ? (size_t)KM_BM * KM_LDD
                                                                                      : (size_t)(KM_BM + KM_BN) * KM_LDS);
}

// One launch of the distance kernel: centre j of group g is c[g * c_gstride + j * d], its squared norm
// cn[g * cn_gstride + j]; the epilogue writes whichever outputs are non-null.
struct KmDist {
  const float* x;
  const double* xn;
  const double* c;
  const double* cn;
  long long c_gstride;
  int m, d, kk, groups, gpc, cn_gstride;
  const int32_t* state;     // non-null: only groups with state[2g] == 0 run
  int32_t* labels;          // [groups, m]
  int* changed;             // [groups]: set when a label differs from the stored one
  double* dist;             // [groups, m] distance to the nearest centre
  double* wmin;             // [groups, m] seeding weights: max(0, dist), min-updated unless wfirst
  int wfirst;
  int32_t* counts;          // [groups, 2, kk]: split at n_eval
  int n_eval;
};

__device__ __forceinline__ bool km_running(const int32_t* state, int g) { return state == nullptr || state[2 * g] == 0; }

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// grid (point tiles, group tiles); 8 warps as 4 (points) x 2 (centres), each 32 x 32 = 4 x 4 DMMA tiles
__global__ void __launch_bounds__(KM_THREADS, 2) km_dist_kernel(const __grid_constant__ KmDist p) {
  extern __shared__ double km_smem[];
  double* As = km_smem;                       // [KM_BM][KM_LDS]  points x k
  double* Bs = km_smem + KM_BM * KM_LDS;      // [KM_BN][KM_LDS]  centres x k
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp & 3, wn = warp >> 2;
  const int m0 = blockIdx.x * KM_BM, g0 = blockIdx.y * p.gpc;
  bool any = false;
  for (int gl = 0; gl < p.gpc && g0 + gl < p.groups; ++gl) any |= km_running(p.state, g0 + gl);
  if (!any) return;

  // staging: points: thread t owns k column t % 32 of rows t / 32 + 8 r; centres: row t / 4, k columns 8 (t % 4) + e
  const int kc = tid & 31, r0 = tid >> 5, nb = tid >> 2, kb = (tid & 3) * 8;
  const double* bsrc = nullptr;
  {
    const int gl = nb / p.kk, g = g0 + gl;
    if (gl < p.gpc && g < p.groups) bsrc = p.c + g * p.c_gstride + (long long)(nb - gl * p.kk) * p.d;
  }
  float ra[KM_BM / 8];
  double rb[8];
  auto load = [&](int k0) {
    const int k = k0 + kc;
#pragma unroll
    for (int r = 0; r < KM_BM / 8; ++r) {
      const int i = m0 + r0 + 8 * r;
      ra[r] = (i < p.m && k < p.d) ? __ldg(p.x + (long long)i * p.d + k) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) rb[e] = (bsrc && k0 + kb + e < p.d) ? __ldg(bsrc + k0 + kb + e) : 0.0;
  };
  auto store = [&]() {
#pragma unroll
    for (int r = 0; r < KM_BM / 8; ++r) As[(r0 + 8 * r) * KM_LDS + kc] = (double)ra[r];
#pragma unroll
    for (int e = 0; e < 8; ++e) Bs[nb * KM_LDS + kb + e] = rb[e];
  };

  double acc[4][4][2];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b][0] = acc[a][b][1] = 0.0;

  const int fr = lane >> 2, fc = lane & 3;
  load(0);
  for (int k0 = 0; k0 < p.d; k0 += KM_BK) {
    __syncthreads();
    store();
    __syncthreads();
    if (k0 + KM_BK < p.d) load(k0 + KM_BK);
#pragma unroll
    for (int kq = 0; kq < KM_BK; kq += 4) {
      double af[4], bf[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        af[t] = As[(wm * 32 + t * 8 + fr) * KM_LDS + kq + fc];
        bf[t] = Bs[(wn * 32 + t * 8 + fr) * KM_LDS + kq + fc];
      }
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) dmma(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
    }
  }
  __syncthreads();

  // epilogue: squared distances into smem, then one thread per (point, group) scans the group's kk columns
  double* D = km_smem;   // [KM_BM][KM_LDD]
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int r = wm * 32 + a * 8 + fr, i = m0 + r;
    const double xn = i < p.m ? p.xn[i] : 0.0;
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = wn * 32 + b * 8 + 2 * fc + h, gl = n / p.kk, g = g0 + gl;
        const double cn = (gl < p.gpc && g < p.groups) ? p.cn[(long long)g * p.cn_gstride + (n - gl * p.kk)] : 0.0;
        D[r * KM_LDD + n] = __dsub_rn(__dadd_rn(xn, cn), __dmul_rn(2.0, acc[a][b][h]));
      }
  }
  __syncthreads();
  for (int q = tid; q < KM_BM * p.gpc; q += KM_THREADS) {
    const int r = q % KM_BM, gl = q / KM_BM, g = g0 + gl, i = m0 + r;
    if (i >= p.m || g >= p.groups || !km_running(p.state, g)) continue;
    const double* row = D + r * KM_LDD + gl * p.kk;
    double best = row[0];
    int lab = 0;
    for (int j = 1; j < p.kk; ++j)
      if (row[j] < best) {
        best = row[j];
        lab = j;
      }
    const long long o = (long long)g * p.m + i;
    if (p.labels) {
      if (p.changed && p.labels[o] != lab) p.changed[g] = 1;
      p.labels[o] = lab;
    }
    if (p.dist) p.dist[o] = best;
    if (p.wmin) {
      const double w = fmax(best, 0.0);
      p.wmin[o] = p.wfirst ? w : fmin(p.wmin[o], w);
    }
    if (p.counts) atomicAdd(p.counts + ((long long)g * 2 + (i >= p.n_eval ? 1 : 0)) * p.kk + lab, 1);
  }
}

// out[r] = sum_c v[r, c]^2 in float64: one warp per row, lane-strided then a fixed shuffle tree
template <typename T>
__global__ void km_sqnorm_kernel(double* __restrict__ out, const T* __restrict__ v, long long rows, int d, int rows_per_group,
                                 const int32_t* state) {
  const long long r = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (r >= rows || !km_running(state, (int)(r / rows_per_group))) return;
  const T* p = v + r * d;
  double s = 0.0;
  for (int c = lane; c < d; c += 32) {
    const double t = (double)p[c];
    s = __fma_rn(t, t, s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
  if (lane == 0) out[r] = s;
}

// k-means++ pick of centre j of every group: grid (groups), KM_THREADS threads.  Copies the point into the centroids
// and stores its squared norm.
__global__ void __launch_bounds__(KM_THREADS) km_pick_kernel(double* __restrict__ c, double* __restrict__ cn,
                                                             const float* __restrict__ x, const double* __restrict__ w,
                                                             const double* __restrict__ uni, int m, int d, int k, int j) {
  __shared__ int s_idx;
  __shared__ double red[KM_THREADS];
  const int g = blockIdx.x;
  if (threadIdx.x == 0) {
    const double u = uni[(long long)g * k + j];
    int idx = (int)fmin(floor(u * m), (double)(m - 1));
    if (j > 0) {
      const double* wg = w + (long long)g * m;
      double tot = 0.0;
#pragma unroll 8
      for (int i = 0; i < m; ++i) tot = __dadd_rn(tot, wg[i]);
      if (tot > 0.0) {
        const double t = __dmul_rn(u, tot);
        double s = 0.0;
        idx = m - 1;
        for (int i = 0; i < m; ++i) {
          s = __dadd_rn(s, wg[i]);
          if (s > t) {
            idx = i;
            break;
          }
        }
      }
    }
    s_idx = idx;
  }
  __syncthreads();
  const float* src = x + (long long)s_idx * d;
  double* dst = c + ((long long)g * k + j) * d;
  double s = 0.0;
  for (int col = threadIdx.x; col < d; col += KM_THREADS) {
    const double v = (double)src[col];
    dst[col] = v;
    s = __fma_rn(v, v, s);
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = KM_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  if (threadIdx.x == 0) cn[(long long)g * k + j] = red[0];
}

// Lloyd update of columns [blockIdx.x * KM_UPD_COLS, +KM_UPD_COLS) of group blockIdx.y: per-cluster sums over the
// points in order (one thread per column, accumulators in smem), means, and the partial squared shift of the chunk.
__global__ void __launch_bounds__(KM_UPD_COLS) km_update_kernel(double* __restrict__ c, double* __restrict__ shift_part,
                                                                const float* __restrict__ x, const int32_t* __restrict__ labels,
                                                                const int32_t* __restrict__ state, int m, int d, int k) {
  extern __shared__ double km_upd[];       // [k][KM_UPD_COLS] sums, then k counts
  __shared__ double red[KM_UPD_COLS];
  const int g = blockIdx.y;
  if (state[2 * g] != 0) return;
  int* cnt = reinterpret_cast<int*>(km_upd + (size_t)k * KM_UPD_COLS);
  const int tid = threadIdx.x, col = blockIdx.x * KM_UPD_COLS + tid;
  for (int j = 0; j < k; ++j) km_upd[j * KM_UPD_COLS + tid] = 0.0;
  for (int j = tid; j < k; j += KM_UPD_COLS) cnt[j] = 0;
  __syncthreads();
  const int32_t* lab = labels + (long long)g * m;
  const float* xc = x + col;
  const bool in = col < d;
  int i = 0;
  for (; i + 4 <= m; i += 4) {
    int l[4];
    float v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      l[u] = __ldg(lab + i + u);
      v[u] = in ? __ldg(xc + (long long)(i + u) * d) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      double* a = km_upd + l[u] * KM_UPD_COLS + tid;
      *a = __dadd_rn(*a, (double)v[u]);
      if (tid == 0) cnt[l[u]]++;
    }
  }
  for (; i < m; ++i) {
    const int l = __ldg(lab + i);
    double* a = km_upd + l * KM_UPD_COLS + tid;
    *a = __dadd_rn(*a, in ? (double)__ldg(xc + (long long)i * d) : 0.0);
    if (tid == 0) cnt[l]++;
  }
  __syncthreads();
  double sh = 0.0;
  if (in)
    for (int j = 0; j < k; ++j) {
      double* cp = c + ((long long)g * k + j) * d + col;
      const double old = *cp;
      const double nw = cnt[j] > 0 ? __ddiv_rn(km_upd[j * KM_UPD_COLS + tid], (double)cnt[j]) : old;
      *cp = nw;
      const double dl = __dsub_rn(nw, old);
      sh = __dadd_rn(sh, __dmul_rn(dl, dl));
    }
  red[tid] = sh;
  __syncthreads();
  for (int h = KM_UPD_COLS / 2; h > 0; h >>= 1) {
    if (tid < h) red[tid] = __dadd_rn(red[tid], red[tid + h]);
    __syncthreads();
  }
  if (tid == 0) shift_part[(long long)g * gridDim.x + blockIdx.x] = red[0];
}

// convergence test of every running group (sklearn _kmeans_single_lloyd: unchanged labels first, then the shift)
__global__ void km_status_kernel(int32_t* __restrict__ state, const int* __restrict__ changed,
                                 const double* __restrict__ shift_part, int groups, int nchunks, double tol) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= groups || state[2 * g] != 0) return;
  const int it = ++state[2 * g + 1];
  double s = 0.0;
  for (int q = 0; q < nchunks; ++q) s = __dadd_rn(s, shift_part[(long long)g * nchunks + q]);
  if (it > 1 && !changed[g])
    state[2 * g] = 2;
  else if (s <= tol)
    state[2 * g] = 1;
}

// inertia[g] = sum_i dist[g, i]: thread-strided, then a fixed tree; grid (groups)
__global__ void __launch_bounds__(KM_THREADS) km_inertia_kernel(double* __restrict__ inertia, const double* __restrict__ dist,
                                                                int m) {
  __shared__ double red[KM_THREADS];
  const double* dg = dist + (long long)blockIdx.x * m;
  double s = 0.0;
  for (int i = threadIdx.x; i < m; i += KM_THREADS) s = __dadd_rn(s, dg[i]);
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = KM_THREADS / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + h]);
    __syncthreads();
  }
  if (threadIdx.x == 0) inertia[blockIdx.x] = red[0];
}

// carves the workspace into 256-byte aligned pieces
struct KmWs {
  char* base;
  size_t off;
  template <typename T>
  T* take(long long n) {
    T* r = reinterpret_cast<T*>(base ? base + off : nullptr);
    off += ((size_t)n * sizeof(T) + 255) / 256 * 256;
    return r;
  }
};

int km_ws(cgan_ctx* ctx, KmWs* w) {
  void* p = nullptr;
  const int rc = cgan_ws(ctx, w->off, &p);
  w->base = static_cast<char*>(p);
  w->off = 0;
  return rc;
}

int km_norms_x(cgan_ctx* ctx, double* xn, const float* x, int m, int d) {
  km_sqnorm_kernel<float><<<cdiv(m, 8), 256, 0, ctx->stream>>>(xn, x, m, d, m, nullptr);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int km_launch_dist(cgan_ctx* ctx, const KmDist& p) {
  CGAN_CUDA(ctx, cudaFuncSetAttribute(km_dist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)km_dist_smem()));
  const dim3 grid(cdiv(p.m, KM_BM), cdiv(p.groups, p.gpc));
  km_dist_kernel<<<grid, KM_THREADS, km_dist_smem(), ctx->stream>>>(p);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

KmDist km_desc(const float* x, const double* xn, const double* c, const double* cn, int m, int d, int k, int groups) {
  KmDist p;
  memset(&p, 0, sizeof(p));
  p.x = x; p.xn = xn; p.c = c; p.cn = cn;
  p.m = m; p.d = d; p.kk = k; p.groups = groups; p.gpc = KM_BN / k;
  p.c_gstride = (long long)k * d; p.cn_gstride = k;
  return p;
}

}  // namespace

#define KM_CHECK_SHAPE(ctx)                                                                                  \
  do {                                                                                                       \
    CGAN_REQUIRE(ctx, k >= 1 && d >= 1 && groups >= 1, "k, d and groups must be >= 1");                     \
    CGAN_REQUIRE(ctx, k <= KM_MAX_K, "k must be <= 64");                                                     \
    CGAN_REQUIRE(ctx, m >= k, "m must be >= k");                                                             \
  } while (0)

int cgan_kmeans_seed(cgan_ctx* ctx, double* centroids, const float* x, int m, int d, int k, int groups,
                     const double* host_uniforms) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, centroids && x && host_uniforms, "null pointer");
  KM_CHECK_SHAPE(ctx);
  for (long long q = 0; q < (long long)groups * k; ++q)
    CGAN_REQUIRE(ctx, host_uniforms[q] >= 0.0 && host_uniforms[q] < 1.0, "uniforms must be in [0, 1)");
  KmWs ws{nullptr, 0};
  ws.take<double>(m);
  ws.take<double>((long long)groups * k);
  ws.take<double>((long long)groups * m);
  ws.take<double>((long long)groups * k);
  int rc = km_ws(ctx, &ws);
  if (rc) return rc;
  double* xn = ws.take<double>(m);
  double* cn = ws.take<double>((long long)groups * k);
  double* w = ws.take<double>((long long)groups * m);
  double* uni = ws.take<double>((long long)groups * k);
  CGAN_CUDA(ctx, cudaMemcpyAsync(uni, host_uniforms, sizeof(double) * groups * k, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = km_norms_x(ctx, xn, x, m, d))) return rc;
  // distances to the newest centre only: one centre per group, KM_BN groups per CTA column
  KmDist p = km_desc(x, xn, centroids, cn, m, d, 1, groups);
  p.c_gstride = (long long)k * d;
  p.cn_gstride = k;
  p.wmin = w;
  for (int j = 0; j < k; ++j) {
    km_pick_kernel<<<groups, KM_THREADS, 0, ctx->stream>>>(centroids, cn, x, w, uni, m, d, k, j);
    CGAN_LAUNCHED(ctx);
    if (j + 1 == k) break;
    p.c = centroids + (long long)j * d;
    p.cn = cn + j;
    p.wfirst = j == 0;
    if ((rc = km_launch_dist(ctx, p))) return rc;
  }
  return CGAN_OK;
}

int cgan_kmeans_lloyd_step(cgan_ctx* ctx, double* centroids, int32_t* labels, int32_t* state, const float* x, int m, int d,
                           int k, int groups, double tol) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, centroids && labels && state && x, "null pointer");
  KM_CHECK_SHAPE(ctx);
  CGAN_REQUIRE(ctx, tol >= 0.0, "tol must be >= 0");
  const int nchunks = cdiv(d, KM_UPD_COLS);
  KmWs ws{nullptr, 0};
  ws.take<double>(m);
  ws.take<double>((long long)groups * k);
  ws.take<int>(groups);
  ws.take<double>((long long)groups * nchunks);
  int rc = km_ws(ctx, &ws);
  if (rc) return rc;
  double* xn = ws.take<double>(m);
  double* cn = ws.take<double>((long long)groups * k);
  int* changed = ws.take<int>(groups);
  double* part = ws.take<double>((long long)groups * nchunks);
  CGAN_CUDA(ctx, cudaMemsetAsync(changed, 0, sizeof(int) * groups, ctx->stream));
  if ((rc = km_norms_x(ctx, xn, x, m, d))) return rc;
  km_sqnorm_kernel<double><<<cdiv((long long)groups * k, 8), 256, 0, ctx->stream>>>(cn, centroids, (long long)groups * k, d, k,
                                                                                      state);
  CGAN_LAUNCHED(ctx);
  KmDist p = km_desc(x, xn, centroids, cn, m, d, k, groups);
  p.state = state;
  p.labels = labels;
  p.changed = changed;
  if ((rc = km_launch_dist(ctx, p))) return rc;
  const size_t smem = sizeof(double) * (size_t)k * KM_UPD_COLS + sizeof(int) * k;
  CGAN_CUDA(ctx, cudaFuncSetAttribute(km_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  km_update_kernel<<<dim3(nchunks, groups), KM_UPD_COLS, smem, ctx->stream>>>(centroids, part, x, labels, state, m, d, k);
  CGAN_LAUNCHED(ctx);
  km_status_kernel<<<cdiv(groups, 128), 128, 0, ctx->stream>>>(state, changed, part, groups, nchunks, tol);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_kmeans_finish(cgan_ctx* ctx, int32_t* labels, double* inertia, int32_t* counts, const double* centroids,
                       const float* x, int m, int d, int k, int groups, int n_eval) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, labels && inertia && counts && centroids && x, "null pointer");
  KM_CHECK_SHAPE(ctx);
  CGAN_REQUIRE(ctx, n_eval >= 0 && n_eval <= m, "n_eval must be in [0, m]");
  KmWs ws{nullptr, 0};
  ws.take<double>(m);
  ws.take<double>((long long)groups * k);
  ws.take<double>((long long)groups * m);
  int rc = km_ws(ctx, &ws);
  if (rc) return rc;
  double* xn = ws.take<double>(m);
  double* cn = ws.take<double>((long long)groups * k);
  double* dist = ws.take<double>((long long)groups * m);
  CGAN_CUDA(ctx, cudaMemsetAsync(counts, 0, sizeof(int32_t) * groups * 2 * k, ctx->stream));
  if ((rc = km_norms_x(ctx, xn, x, m, d))) return rc;
  km_sqnorm_kernel<double><<<cdiv((long long)groups * k, 8), 256, 0, ctx->stream>>>(cn, centroids, (long long)groups * k, d, k,
                                                                                      nullptr);
  CGAN_LAUNCHED(ctx);
  KmDist p = km_desc(x, xn, centroids, cn, m, d, k, groups);
  p.labels = labels;
  p.dist = dist;
  p.counts = counts;
  p.n_eval = n_eval;
  if ((rc = km_launch_dist(ctx, p))) return rc;
  km_inertia_kernel<<<groups, KM_THREADS, 0, ctx->stream>>>(inertia, dist, m);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}
