// Exact-fp32 gather-GEMM family: conv2d fwd / dgrad / wgrad (implicit GEMM over NHWC + HWIO,
// TF SAME padding, strides, fused zero-insertion upsampling) and plain/batched row-major GEMM.
// This is math_mode 0: the bit-faithful fp32 contraction every shape can fall back to and the
// on-device yard-stick for the tensor-core path (conv_tc.cu).
//
// Replaces: tf.nn.conv2d (arch_ops.py:568), its autodiff Conv2DBackpropInput/Filter,
// tf.nn.conv2d_transpose (arch_ops.py:588-589), resnet_ops.unpool+conv (resnet_ops.py:122-130),
// tf.matmul (arch_ops.py:548, 744, 753).
#include "common.cuh"

namespace {

enum { M_GEMM = 0, M_FWD = 1, M_DGRAD = 2, M_WGRAD = 3 };

struct GP {
  int M, N, K;
  const float* A;
  const float* B;
  float* C;
  const float* bias;
  float alpha, beta;
  int lda, ldb, ldc, ta, tb;
  long long sA, sB, sC;   // batch strides (GEMM) — blockIdx.z = batch
  cgan_conv_desc d;
  int vh, vw;             // virtual (post-upsample) input size
  int splits, k_per_split;  // split-K (WGRAD) — blockIdx.z = split; partial results to `C` + z*M*N
  int vecA, vecB;         // host-verified: 8-wide vector loads are legal
  int relu;               // fused ReLU (inference-only callers)
};

constexpr int BM = 128, BK = 16, NT = 256;

struct Pix { int n, y, x; };

__device__ __forceinline__ Pix decode_pix(int m, int hh, int ww) {
  Pix p;
  p.x = m % ww;
  int t = m / ww;
  p.y = t % hh;
  p.n = t / hh;
  return p;
}

// offset of x[n, ih, iw, 0] for output pixel (oh,ow) and tap (kh,kw); -1 when the tap reads padding / inserted zeros
__device__ __forceinline__ long long in_offset(const GP& p, int n, int oh, int ow, int kh, int kw) {
  const cgan_conv_desc& d = p.d;
  int vh = oh * d.stride + kh - d.pad_t, vw = ow * d.stride + kw - d.pad_l;
  if (vh < 0 || vw < 0 || vh >= p.vh || vw >= p.vw) return -1;
  if (d.upsample) {
    if ((vh | vw) & 1) return -1;
    vh >>= 1;
    vw >>= 1;
  }
  return (((long long)n * d.h + vh) * d.w + vw) * d.cin;
}

// offset of dy[n, oh, ow, 0] contributing to input pixel (ih,iw) through tap (kh,kw); -1 if none
__device__ __forceinline__ long long out_offset(const GP& p, int n, int ih, int iw, int kh, int kw) {
  const cgan_conv_desc& d = p.d;
  int vh = d.upsample ? 2 * ih : ih, vw = d.upsample ? 2 * iw : iw;
  int th = vh + d.pad_t - kh, tw = vw + d.pad_l - kw;
  if (th < 0 || tw < 0) return -1;
  int oh = th / d.stride, ow = tw / d.stride;
  if (oh * d.stride != th || ow * d.stride != tw) return -1;
  if (oh >= d.oh || ow >= d.ow) return -1;
  return (((long long)n * d.oh + oh) * d.ow + ow) * d.cout;
}

template <int MODE>
__device__ __forceinline__ float a_elem(const GP& p, int m, int k) {
  if (m >= p.M || k >= p.K) return 0.f;
  if (MODE == M_GEMM) return p.ta ? p.A[(long long)k * p.lda + m] : p.A[(long long)m * p.lda + k];
  const cgan_conv_desc& d = p.d;
  if (MODE == M_FWD) {
    Pix o = decode_pix(m, d.oh, d.ow);
    int ci = k % d.cin, tap = k / d.cin;
    long long off = in_offset(p, o.n, o.y, o.x, tap / d.kw, tap % d.kw);
    return off < 0 ? 0.f : p.A[off + ci];
  }
  if (MODE == M_DGRAD) {
    Pix i = decode_pix(m, d.h, d.w);
    int co = k % d.cout, tap = k / d.cout;
    long long off = out_offset(p, i.n, i.y, i.x, tap / d.kw, tap % d.kw);
    return off < 0 ? 0.f : p.A[off + co];
  }
  // WGRAD: m = (tap, ci), k = output pixel
  Pix o = decode_pix(k, d.oh, d.ow);
  int ci = m % d.cin, tap = m / d.cin;
  long long off = in_offset(p, o.n, o.y, o.x, tap / d.kw, tap % d.kw);
  return off < 0 ? 0.f : p.A[off + ci];
}

template <int MODE>
__device__ __forceinline__ float b_elem(const GP& p, int k, int n) {
  if (k >= p.K || n >= p.N) return 0.f;
  if (MODE == M_GEMM) return p.tb ? p.B[(long long)n * p.ldb + k] : p.B[(long long)k * p.ldb + n];
  const cgan_conv_desc& d = p.d;
  if (MODE == M_FWD) return p.B[(long long)k * d.cout + n];
  if (MODE == M_DGRAD) {
    int co = k % d.cout, tap = k / d.cout;
    return p.B[((long long)tap * d.cin + n) * d.cout + co];
  }
  return p.B[(long long)k * d.cout + n];   // WGRAD: dy[pixel, co]
}

__device__ __forceinline__ void ld8(const float* ptr, float (&v)[8]) {
  float4 a = __ldg(reinterpret_cast<const float4*>(ptr));
  float4 b = __ldg(reinterpret_cast<const float4*>(ptr) + 1);
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
__device__ __forceinline__ void zero8(float (&v)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = 0.f;
}

// 8 A elements: AKF ? (m, k..k+7) : (m..m+7, k).  k and m are multiples of 8 relative to tile origins.
template <int MODE, bool AKF>
__device__ __forceinline__ void load_a8(const GP& p, int m, int k, float (&v)[8]) {
  if (p.vecA) {
    const cgan_conv_desc& d = p.d;
    if (MODE == M_GEMM) {
      if (AKF) {
        if (m < p.M && k + 8 <= p.K) { ld8(p.A + (long long)m * p.lda + k, v); return; }
      } else {
        if (k < p.K && m + 8 <= p.M) { ld8(p.A + (long long)k * p.lda + m, v); return; }
      }
    } else if (MODE == M_FWD) {       // cin % 8 == 0: the 8 k share one tap
      if (m >= p.M || k >= p.K) { zero8(v); return; }
      Pix o = decode_pix(m, d.oh, d.ow);
      int ci = k % d.cin, tap = k / d.cin;
      long long off = in_offset(p, o.n, o.y, o.x, tap / d.kw, tap % d.kw);
      if (off < 0) zero8(v); else ld8(p.A + off + ci, v);
      return;
    } else if (MODE == M_DGRAD) {     // cout % 8 == 0
      if (m >= p.M || k >= p.K) { zero8(v); return; }
      Pix i = decode_pix(m, d.h, d.w);
      int co = k % d.cout, tap = k / d.cout;
      long long off = out_offset(p, i.n, i.y, i.x, tap / d.kw, tap % d.kw);
      if (off < 0) zero8(v); else ld8(p.A + off + co, v);
      return;
    } else {                          // WGRAD, m-fast: cin % 8 == 0, the 8 m share one tap
      if (m >= p.M || k >= p.K) { zero8(v); return; }
      Pix o = decode_pix(k, d.oh, d.ow);
      int ci = m % d.cin, tap = m / d.cin;
      long long off = in_offset(p, o.n, o.y, o.x, tap / d.kw, tap % d.kw);
      if (off < 0) zero8(v); else ld8(p.A + off + ci, v);
      return;
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = AKF ? a_elem<MODE>(p, m, k + j) : a_elem<MODE>(p, m + j, k);
}

// E B elements: BKF ? (k..k+E-1, n) : (k, n..n+E-1)
template <int MODE, bool BKF, int E>
__device__ __forceinline__ void load_b(const GP& p, int k, int n, float (&v)[8]) {
  if (E == 8 && p.vecB) {
    const cgan_conv_desc& d = p.d;
    if (MODE == M_GEMM) {
      if (BKF) {
        if (n < p.N && k + 8 <= p.K) { ld8(p.B + (long long)n * p.ldb + k, v); return; }
      } else {
        if (k < p.K && n + 8 <= p.N) { ld8(p.B + (long long)k * p.ldb + n, v); return; }
      }
    } else if (MODE == M_DGRAD) {     // k-fast: cout % 8 == 0
      if (k >= p.K || n >= p.N) { zero8(v); return; }
      int co = k % d.cout, tap = k / d.cout;
      ld8(p.B + ((long long)tap * d.cin + n) * d.cout + co, v);
      return;
    } else {                          // FWD / WGRAD: rows of [K, cout], cout % 8 == 0
      if (k < p.K && n + 8 <= p.N) { ld8(p.B + (long long)k * d.cout + n, v); return; }
    }
  }
#pragma unroll
  for (int j = 0; j < E; ++j) v[j] = BKF ? b_elem<MODE>(p, k + j, n) : b_elem<MODE>(p, k, n + j);
}

template <int MODE, bool AKF, bool BKF, int BN>
__global__ void __launch_bounds__(NT, 2) gather_gemm_kernel(GP p) {
  constexpr int TN = BN / 16;          // columns per thread: 8 (two groups of 4) or 2
  constexpr int EB = BN * BK / NT;     // B elements loaded per thread: 8 or 2
  __shared__ __align__(16) float As[2][BK][BM + 4];
  __shared__ __align__(16) float Bs[2][BK][BN + 4];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;   // M tiles on x: up to 2^31-1 of them

  int kbeg = 0, kend = p.K;
  if (MODE == M_GEMM) {
    p.A += (long long)blockIdx.z * p.sA;
    p.B += (long long)blockIdx.z * p.sB;
    p.C += (long long)blockIdx.z * p.sC;
  } else if (p.splits > 1) {
    kbeg = blockIdx.z * p.k_per_split;
    kend = min(p.K, kbeg + p.k_per_split);
    p.C += (long long)blockIdx.z * p.M * p.N;
  }

  // per-thread load coordinates inside a tile
  const int a_m = AKF ? (tid >> 1) : (tid & 15) * 8;
  const int a_k = AKF ? (tid & 1) * 8 : (tid >> 4);
  int b_k, b_n;
  if (BKF) {
    constexpr int TPR = BK / EB;       // threads per n-row
    b_n = tid / TPR;
    b_k = (tid % TPR) * EB;
  } else {
    constexpr int TPR = BN / EB;       // threads per k-row
    b_k = tid / TPR;
    b_n = (tid % TPR) * EB;
  }

  float ra[8], rb[8];
  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  auto gload = [&](int k0) {
    load_a8<MODE, AKF>(p, m0 + a_m, k0 + a_k, ra);
    // a split must not read past its own K range
    if (kend < p.K) {
      if (AKF) {
#pragma unroll
        for (int j = 0; j < 8; ++j) if (k0 + a_k + j >= kend) ra[j] = 0.f;
      } else if (k0 + a_k >= kend) {
        zero8(ra);
      }
    }
    load_b<MODE, BKF, EB>(p, k0 + b_k, n0 + b_n, rb);
    if (kend < p.K) {
      if (BKF) {
#pragma unroll
        for (int j = 0; j < EB; ++j) if (k0 + b_k + j >= kend) rb[j] = 0.f;
      } else if (k0 + b_k >= kend) {
#pragma unroll
        for (int j = 0; j < EB; ++j) rb[j] = 0.f;
      }
    }
  };
  auto sstore = [&](int buf) {
    if (AKF) {
#pragma unroll
      for (int j = 0; j < 8; ++j) As[buf][a_k + j][a_m] = ra[j];
    } else {
      *reinterpret_cast<float4*>(&As[buf][a_k][a_m]) = make_float4(ra[0], ra[1], ra[2], ra[3]);
      *reinterpret_cast<float4*>(&As[buf][a_k][a_m + 4]) = make_float4(ra[4], ra[5], ra[6], ra[7]);
    }
    if (BKF) {
#pragma unroll
      for (int j = 0; j < EB; ++j) Bs[buf][b_k + j][b_n] = rb[j];
    } else if constexpr (EB == 8) {
      *reinterpret_cast<float4*>(&Bs[buf][b_k][b_n]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
      *reinterpret_cast<float4*>(&Bs[buf][b_k][b_n + 4]) = make_float4(rb[4], rb[5], rb[6], rb[7]);
    } else {
#pragma unroll
      for (int j = 0; j < EB; ++j) Bs[buf][b_k][b_n + j] = rb[j];
    }
  };

  const int ntiles = (kend - kbeg + BK - 1) / BK;
  if (ntiles > 0) {
    gload(kbeg);
    sstore(0);
  }
  __syncthreads();
  for (int t = 0; t < ntiles; ++t) {
    const int buf = t & 1;
    if (t + 1 < ntiles) gload(kbeg + (t + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      float a[8], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w;
      a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      if constexpr (TN == 8) {
        float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
        float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][(BN / 2) + tx * 4]);
        b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
        b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
      } else {
        float2 b0 = *reinterpret_cast<const float2*>(&Bs[buf][kk][tx * 2]);
        b[0] = b0.x; b[1] = b0.y;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (t + 1 < ntiles) sstore(buf ^ 1);
    __syncthreads();
  }

  // epilogue
  const bool partial = (MODE != M_GEMM) && p.splits > 1;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      int n;
      if constexpr (TN == 8) n = n0 + (j < 4 ? tx * 4 + j : (BN / 2) + tx * 4 + (j - 4));
      else n = n0 + tx * 2 + j;
      if (n >= p.N) continue;
      long long idx = (long long)m * p.ldc + n;
      float r = acc[i][j];
      if (!partial) {
        r *= p.alpha;
        if (p.beta != 0.f) r += p.beta * p.C[idx];
        if (p.bias) r += p.bias[n];
        if (p.relu) r = fmaxf(r, 0.f);
      }
      p.C[idx] = r;
    }
  }
}

__global__ void splitk_reduce_kernel(float* __restrict__ out, const float* __restrict__ part, long long n, int splits) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int z = 0; z < splits; ++z) s += part[(long long)z * n + i];
  out[i] = s;
}

template <int MODE, bool AKF, bool BKF>
int launch(cgan_ctx* ctx, const GP& p, int gz) {
  if (p.M <= 0 || p.N <= 0) return CGAN_OK;
  if (p.N > 32) {
    dim3 grid(cdiv(p.M, BM), cdiv(p.N, 128), gz);
    gather_gemm_kernel<MODE, AKF, BKF, 128><<<grid, NT, 0, ctx->stream>>>(p);
  } else {
    dim3 grid(cdiv(p.M, BM), cdiv(p.N, 32), gz);
    gather_gemm_kernel<MODE, AKF, BKF, 32><<<grid, NT, 0, ctx->stream>>>(p);
  }
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int check_desc(cgan_ctx* ctx, const cgan_conv_desc* d) {
  CGAN_REQUIRE(ctx, d != nullptr, "null descriptor");
  CGAN_REQUIRE(ctx, d->n > 0 && d->h > 0 && d->w > 0 && d->cin > 0 && d->cout > 0, "non-positive tensor dims");
  CGAN_REQUIRE(ctx, d->kh > 0 && d->kw > 0 && d->stride > 0 && d->oh > 0 && d->ow > 0, "bad kernel/stride/output dims");
  CGAN_REQUIRE(ctx, d->pad_t >= 0 && d->pad_l >= 0, "negative padding");
  CGAN_REQUIRE(ctx, (long long)d->n * d->oh * d->ow < (1ll << 31) && (long long)d->n * d->h * d->w < (1ll << 31),
               "pixel count exceeds int32");
  return CGAN_OK;
}

GP conv_gp(const cgan_conv_desc* d) {
  GP p;
  memset(&p, 0, sizeof(p));
  p.d = *d;
  p.vh = d->upsample ? 2 * d->h : d->h;
  p.vw = d->upsample ? 2 * d->w : d->w;
  p.alpha = 1.f;
  p.splits = 1;
  return p;
}

}  // namespace

int cgan_conv2d_fwd_simt(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, float* y,
                         int relu, int ldy) {
  int rc = check_desc(ctx, d);
  if (rc) return rc;
  GP p = conv_gp(d);
  p.M = d->n * d->oh * d->ow;
  p.N = d->cout;
  p.K = d->kh * d->kw * d->cin;
  p.A = x; p.B = w; p.C = y; p.bias = bias;
  p.relu = relu;
  p.ldc = ldy;
  p.vecA = (d->cin % 8 == 0) && al16(x);
  p.vecB = (d->cout % 8 == 0) && al16(w);
  return launch<M_FWD, true, false>(ctx, p, 1);
}

int cgan_conv2d_dgrad_simt(cgan_ctx* ctx, const cgan_conv_desc* d, const float* dy, const float* w, float* dx) {
  int rc = check_desc(ctx, d);
  if (rc) return rc;
  GP p = conv_gp(d);
  p.M = d->n * d->h * d->w;
  p.N = d->cin;
  p.K = d->kh * d->kw * d->cout;
  p.A = dy; p.B = w; p.C = dx;
  p.ldc = d->cin;
  p.vecA = (d->cout % 8 == 0) && al16(dy);
  p.vecB = (d->cout % 8 == 0) && al16(w);
  return launch<M_DGRAD, true, true>(ctx, p, 1);
}

int cgan_conv2d_wgrad_simt(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, float* dw) {
  if (!ctx) return CGAN_ERR_ARG;
  int rc = check_desc(ctx, d);
  if (rc) return rc;
  CGAN_REQUIRE(ctx, x && dy && dw, "null pointer");
  GP p = conv_gp(d);
  p.M = d->kh * d->kw * d->cin;
  p.N = d->cout;
  p.K = d->n * d->oh * d->ow;
  p.A = x; p.B = dy;
  p.ldc = d->cout;
  p.vecA = (d->cin % 8 == 0) && al16(x);
  p.vecB = (d->cout % 8 == 0) && al16(dy);
  // split-K so that the (tap,cin) x cout grid fills the SMs about four times over
  long long tiles = (long long)cdiv(p.M, BM) * cdiv(p.N, p.N > 32 ? 128 : 32);
  int ktiles = cdiv(p.K, BK);
  int splits = (int)((4ll * ctx->num_sms + tiles - 1) / tiles);
  if (splits > ktiles) splits = ktiles;
  if (splits > 512) splits = 512;
  if (splits < 1) splits = 1;
  int tiles_per_split = cdiv(ktiles, splits);
  splits = cdiv(ktiles, tiles_per_split);
  p.splits = splits;
  p.k_per_split = tiles_per_split * BK;
  if (splits == 1) {
    p.C = dw;
    return launch<M_WGRAD, false, false>(ctx, p, 1);
  }
  void* ws = nullptr;
  long long mn = (long long)p.M * p.N;
  rc = cgan_ws(ctx, (size_t)splits * mn * sizeof(float), &ws);
  if (rc) return rc;
  p.C = reinterpret_cast<float*>(ws);
  rc = launch<M_WGRAD, false, false>(ctx, p, splits);
  if (rc) return rc;
  return cgan_splitk_reduce(ctx, dw, p.C, mn, splits);
}

int cgan_splitk_reduce(cgan_ctx* ctx, float* out, const float* part, long long n, int splits) {
  splitk_reduce_kernel<<<cdiv(n, 256), 256, 0, ctx->stream>>>(out, part, n, splits);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_gemm_batched_simt(cgan_ctx* ctx, int ta, int tb, int m, int n, int k, float alpha, const float* a, int lda,
                      int64_t sa, const float* b, int ldb, int64_t sb, float beta, float* c, int ldc, int64_t sc,
                      int batch) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, m >= 0 && n >= 0 && k >= 0 && batch >= 0, "negative size");
  CGAN_REQUIRE(ctx, a && b && c, "null pointer");
  CGAN_REQUIRE(ctx, batch <= 65535, "batch exceeds grid.z");
  if (m == 0 || n == 0 || batch == 0) return CGAN_OK;
  GP p;
  memset(&p, 0, sizeof(p));
  p.M = m; p.N = n; p.K = k;
  p.A = a; p.B = b; p.C = c;
  p.alpha = alpha; p.beta = beta;
  p.lda = lda; p.ldb = ldb; p.ldc = ldc; p.ta = ta; p.tb = tb;
  p.sA = sa; p.sB = sb; p.sC = sc;
  p.splits = 1;
  p.vecA = al16(a) && lda % 4 == 0 && sa % 4 == 0;
  p.vecB = al16(b) && ldb % 4 == 0 && sb % 4 == 0;
  if (!ta && !tb) return launch<M_GEMM, true, false>(ctx, p, batch);
  if (ta && !tb) return launch<M_GEMM, false, false>(ctx, p, batch);
  if (!ta && tb) return launch<M_GEMM, true, true>(ctx, p, batch);
  return launch<M_GEMM, false, true>(ctx, p, batch);
}

