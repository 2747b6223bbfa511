// Fractal dimension of a generated set (metrics/fractal_dimension.py:39-97): the float64 Euclidean distances of every
// sample to the seed samples, their range, and the number of distances below each bin edge.
//
// The distances are direct differences, not the ||x||^2 + ||s||^2 - 2 x.s expansion: every seed is itself a sample, so
// its self-distance must be exactly 0, and the smallest non-zero distance anchors every bin edge; the expansion cancels
// for near-duplicates.  fd_dist_kernel is a register-blocked SIMT "difference GEMM" on the FP64 pipe: a 64-row x 64-seed
// tile per CTA, 4 x 4 outputs per thread, fp32 values scaled in fp32 and converted to float64 once as they are staged in
// shared memory (the difference of two fp32 values is then exact in float64), squares accumulated with a float64 FMA.
//
// A row's bits depend on d only: D is cut into fixed slices of FD_SLICE columns, each summed sequentially in column
// order by one CTA, and the slices' partial sums are added in slice order.  So a row does not depend on the number of
// rows, on the other rows of the call or on the call's position in a run; the slices let a batch of 256 rows x 100 seeds
// at 128^2 x 3 still spread over every SM.
//
// fd_range and fd_counts are exact and order-free: min / max on the bit patterns of non-negative doubles, and integer
// histograms over the bin edges followed by a prefix sum.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int FD_BM = 64, FD_BN = 64, FD_BK = 32, FD_THREADS = 256;
constexpr int FD_LD = FD_BM + 1;                       // smem row stride (doubles) of the staged [k][row] tiles
constexpr int FD_SLICE = 2048;                         // D columns per slice: a multiple of FD_BK
constexpr long long FD_PART_BYTES = 64ll << 20;        // partial sums of one launch at most
constexpr int FD_MAX_EDGES = 8192;
constexpr int FD_SCAN_THREADS = 1024;

static_assert(FD_SLICE % FD_BK == 0, "a slice holds whole k stages");

// grid (row tiles, seed tiles, slices); 16 x 16 threads, thread (tx, ty) owns rows ty + 16 p and seeds tx + 16 q.
// part == nullptr: one slice, out[i, j] = sqrt(sum) directly; else part[z, i, j] = the sum over slice z.
__global__ void __launch_bounds__(FD_THREADS) fd_dist_kernel(double* __restrict__ out, double* __restrict__ part,
                                                             const float* __restrict__ x, int n,
                                                             const float* __restrict__ sd, int s, int d, float scale) {
  __shared__ double As[FD_BK * FD_LD];
  __shared__ double Bs[FD_BK * FD_LD];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int i0 = blockIdx.x * FD_BM, j0 = blockIdx.y * FD_BN;
  const int k_lo = blockIdx.z * FD_SLICE, k_hi = min(d, k_lo + FD_SLICE);

  // staging: thread t loads column t % 32 of rows (and seeds) t / 32 + 8 r: one coalesced 128-byte row piece per warp
  const int kc = tid & 31, r0 = tid >> 5;
  float ra[FD_BM / 8], rb[FD_BN / 8];
  auto load = [&](int k0) {
    const int k = k0 + kc;
#pragma unroll
    for (int r = 0; r < FD_BM / 8; ++r) {
      const int i = i0 + r0 + 8 * r;
      ra[r] = (i < n && k < k_hi) ? __ldg(x + (long long)i * d + k) : 0.f;
    }
#pragma unroll
    for (int r = 0; r < FD_BN / 8; ++r) {
      const int j = j0 + r0 + 8 * r;
      rb[r] = (j < s && k < k_hi) ? __ldg(sd + (long long)j * d + k) : 0.f;
    }
  };
  // padding (k >= k_hi) is 0 on both sides: its difference is 0 and fma(0, 0, acc) == acc
  auto store = [&]() {
#pragma unroll
    for (int r = 0; r < FD_BM / 8; ++r) As[kc * FD_LD + r0 + 8 * r] = (double)__fmul_rn(scale, ra[r]);
#pragma unroll
    for (int r = 0; r < FD_BN / 8; ++r) Bs[kc * FD_LD + r0 + 8 * r] = (double)__fmul_rn(scale, rb[r]);
  };

  double acc[4][4];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[p][q] = 0.0;

  load(k_lo);
  for (int k0 = k_lo; k0 < k_hi; k0 += FD_BK) {
    __syncthreads();
    store();
    __syncthreads();
    if (k0 + FD_BK < k_hi) load(k0 + FD_BK);
#pragma unroll 8
    for (int kk = 0; kk < FD_BK; ++kk) {
      double a[4], b[4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        a[t] = As[kk * FD_LD + ty + 16 * t];      // two distinct rows per warp: broadcast
        b[t] = Bs[kk * FD_LD + tx + 16 * t];      // 16 consecutive seeds per warp
      }
#pragma unroll
      for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const double t = __dsub_rn(a[p], b[q]);
          acc[p][q] = __fma_rn(t, t, acc[p][q]);
        }
    }
  }

#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int i = i0 + ty + 16 * p;
    if (i >= n) continue;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int j = j0 + tx + 16 * q;
      if (j >= s) continue;
      if (part)
        part[((long long)blockIdx.z * n + i) * s + j] = acc[p][q];
      else
        out[(long long)i * s + j] = __dsqrt_rn(acc[p][q]);
    }
  }
}

// out[q] = sqrt(part[0, q] + part[1, q] + ... + part[nslices - 1, q]), added in slice order
__global__ void fd_reduce_kernel(double* __restrict__ out, const double* __restrict__ part, long long count, int nslices) {
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < count; q += (long long)gridDim.x * blockDim.x) {
    double v = part[q];
    for (int z = 1; z < nslices; ++z) v = __dadd_rn(v, part[(long long)z * count + q]);
    out[q] = __dsqrt_rn(v);
  }
}

// For non-negative doubles (and +NaN, above +inf) the bit patterns order like the values.
__global__ void fd_range_init_kernel(unsigned long long* r) {
  r[0] = 0x7ff0000000000000ull;      // +inf: no non-zero distance seen
  r[1] = 0ull;
}

__global__ void fd_range_kernel(unsigned long long* __restrict__ r, const double* __restrict__ dist, long long count) {
  unsigned long long lo = 0x7ff0000000000000ull, hi = 0ull;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < count; q += (long long)gridDim.x * blockDim.x) {
    const double v = dist[q];
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    if (v > 0.0 && b < lo) lo = b;
    if (b > hi) hi = b;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMin(r, lo);
    atomicMax(r + 1, hi);
  }
}

// hist[b] += #{dist < edges[b]} - #{dist < edges[b - 1]}: b = the first edge above the distance (upper bound), so a
// distance on an edge counts for the next edge only; NaN lands in bin nedges, which no count includes
__global__ void __launch_bounds__(256) fd_hist_kernel(unsigned long long* __restrict__ hist, const double* __restrict__ dist,
                                                      long long count, const double* __restrict__ edges, int nedges) {
  extern __shared__ double fd_edges[];
  unsigned* h = reinterpret_cast<unsigned*>(fd_edges + nedges);
  for (int t = threadIdx.x; t < nedges; t += blockDim.x) fd_edges[t] = edges[t];
  for (int t = threadIdx.x; t <= nedges; t += blockDim.x) h[t] = 0u;
  __syncthreads();
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < count; q += (long long)gridDim.x * blockDim.x) {
    const double v = dist[q];
    int lo = 0, hi = nedges;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (fd_edges[mid] > v)
        hi = mid;
      else
        lo = mid + 1;
    }
    atomicAdd(h + lo, 1u);
  }
  __syncthreads();
  for (int t = threadIdx.x; t <= nedges; t += blockDim.x)
    if (h[t]) atomicAdd(hist + t, (unsigned long long)h[t]);
}

// counts[j] = hist[0] + ... + hist[j]: one block, a contiguous chunk of bins per thread
__global__ void __launch_bounds__(FD_SCAN_THREADS) fd_scan_kernel(int64_t* __restrict__ counts,
                                                                  const unsigned long long* __restrict__ hist, int nedges) {
  __shared__ unsigned long long base[FD_SCAN_THREADS];
  const int per = (nedges + FD_SCAN_THREADS - 1) / FD_SCAN_THREADS;
  const int b0 = min(nedges, threadIdx.x * per), b1 = min(nedges, b0 + per);
  unsigned long long s = 0;
  for (int b = b0; b < b1; ++b) s += hist[b];
  base[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long run = 0;
    for (int t = 0; t < FD_SCAN_THREADS; ++t) {
      const unsigned long long v = base[t];
      base[t] = run;
      run += v;
    }
  }
  __syncthreads();
  s = base[threadIdx.x];
  for (int b = b0; b < b1; ++b) {
    s += hist[b];
    counts[b] = (int64_t)s;
  }
}

}  // namespace

int cgan_fd_distances(cgan_ctx* ctx, double* out, const float* x, int n, const float* seeds, int s, int d, float scale) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, out && x && seeds, "null pointer");
  CGAN_REQUIRE(ctx, n >= 1 && s >= 1 && d >= 1, "n, s and d must be >= 1");
  CGAN_REQUIRE(ctx, cdiv(d, FD_SLICE) <= 65535, "d must be <= 65535 * 2048");
  CGAN_REQUIRE(ctx, isfinite(scale), "scale must be finite");
  const int nslices = cdiv(d, FD_SLICE);
  const dim3 block(FD_THREADS);
  if (nslices == 1) {
    fd_dist_kernel<<<dim3(cdiv(n, FD_BM), cdiv(s, FD_BN), 1), block, 0, ctx->stream>>>(out, nullptr, x, n, seeds, s, d,
                                                                                      scale);
    CGAN_LAUNCHED(ctx);
    return CGAN_OK;
  }
  // rows per launch: whole row tiles whose partial sums fit FD_PART_BYTES (row chunks do not change a row's bits)
  long long rows = FD_PART_BYTES / ((long long)nslices * s * (long long)sizeof(double)) / FD_BM * FD_BM;
  rows = rows < FD_BM ? FD_BM : rows;
  rows = rows > n ? n : rows;
  void* ws = nullptr;
  int rc = cgan_ws(ctx, (size_t)nslices * rows * s * sizeof(double), &ws);
  if (rc) return rc;
  double* part = static_cast<double*>(ws);
  for (long long r0 = 0; r0 < n; r0 += rows) {
    const int nr = (int)(n - r0 < rows ? n - r0 : rows);
    fd_dist_kernel<<<dim3(cdiv(nr, FD_BM), cdiv(s, FD_BN), nslices), block, 0, ctx->stream>>>(
        nullptr, part, x + r0 * d, nr, seeds, s, d, scale);
    CGAN_LAUNCHED(ctx);
    const long long count = (long long)nr * s;
    fd_reduce_kernel<<<ew_grid(ctx, count), 256, 0, ctx->stream>>>(out + r0 * s, part, count, nslices);
    CGAN_LAUNCHED(ctx);
  }
  return CGAN_OK;
}

int cgan_fd_range(cgan_ctx* ctx, double* out2, const double* dist, int64_t count) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, out2 && dist, "null pointer");
  CGAN_REQUIRE(ctx, count >= 1, "count must be >= 1");
  unsigned long long* r = reinterpret_cast<unsigned long long*>(out2);
  fd_range_init_kernel<<<1, 1, 0, ctx->stream>>>(r);
  CGAN_LAUNCHED(ctx);
  fd_range_kernel<<<ew_grid(ctx, count), 256, 0, ctx->stream>>>(r, dist, count);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_fd_counts(cgan_ctx* ctx, int64_t* counts, const double* dist, int64_t count, const double* edges, int nedges) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, counts && dist && edges, "null pointer");
  CGAN_REQUIRE(ctx, count >= 1, "count must be >= 1");
  CGAN_REQUIRE(ctx, nedges >= 1 && nedges <= FD_MAX_EDGES, "nedges must be in [1, 8192]");
  void* ws = nullptr;
  int rc = cgan_ws(ctx, sizeof(unsigned long long) * (nedges + 1), &ws);
  if (rc) return rc;
  unsigned long long* hist = static_cast<unsigned long long*>(ws);
  CGAN_CUDA(ctx, cudaMemsetAsync(hist, 0, sizeof(unsigned long long) * (nedges + 1), ctx->stream));
  const size_t smem = sizeof(double) * nedges + sizeof(unsigned) * (nedges + 1);
  CGAN_CUDA(ctx, cudaFuncSetAttribute(fd_hist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int grid = min(ew_grid(ctx, count), 4 * ctx->num_sms);   // each CTA first loads the edges: fewer, longer CTAs
  fd_hist_kernel<<<grid, 256, smem, ctx->stream>>>(hist, dist, count, edges, nedges);
  CGAN_LAUNCHED(ctx);
  fd_scan_kernel<<<1, FD_SCAN_THREADS, 0, ctx->stream>>>(counts, hist, nedges);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}
