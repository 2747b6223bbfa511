// Filter gradients of "thin" convolutions — the image-side layers of every architecture (3 input channels in the
// discriminator's first block, 3 output channels in the generator's last conv).  As GEMMs they are 27 x Cout x pixels
// or (9*Cin) x 3 x pixels: far too skinny for a 128-wide tensor-core tile and purely HBM/L2-bound, so they get
// streaming fp32 kernels: each CTA walks a contiguous range of output pixels, keeps the whole dW tile in registers,
// reads dY (resp. X) exactly once with coalesced 128-byte rows, and writes one partial tile; partials are summed in a
// fixed order (deterministic).  Replaces TF Conv2DBackpropFilter for these shapes (arch_ops.py:568 autodiff).
#include "common.cuh"

namespace {

constexpr int THIN_MAX_M = 36;    // taps * cin  (3x3x4)
constexpr int THIN_PB = 32;       // pixels staged per batch

struct ThinParams {
  cgan_conv_desc d;
  int vh, vw;
  long long npix;                 // n * oh * ow
  long long pix_per_block;
};

// pixel index -> (image, row, column) of the output grid.  The hosts below only launch with npix < 2^31, so this is
// 32-bit unsigned arithmetic (a 64-bit division costs ~10x as many instructions and dominated the staging loops).
__device__ __forceinline__ void thin_pixel(long long pix64, const cgan_conv_desc& d, int& n, int& oh, int& ow) {
  const unsigned pix = (unsigned)pix64;
  const unsigned t = pix / (unsigned)d.ow;
  ow = (int)(pix - t * (unsigned)d.ow);
  const unsigned nn = t / (unsigned)d.oh;
  oh = (int)(t - nn * (unsigned)d.oh);
  n = (int)nn;
}

__device__ __forceinline__ long long thin_in_offset(const ThinParams& p, int n, int oh, int ow, int kh, int kw) {
  const cgan_conv_desc& d = p.d;
  int vh = oh * d.stride + kh - d.pad_t, vw = ow * d.stride + kw - d.pad_l;
  if (vh < 0 || vw < 0 || vh >= p.vh || vw >= p.vw) return -1;
  if (d.upsample) {
    if ((vh | vw) & 1) return -1;
    vh >>= 1; vw >>= 1;
  }
  return (((long long)n * d.h + vh) * d.w + vw) * d.cin;
}

// Cin <= 4: thread = output channel; acc[m] over m = (tap, ci)
template <int M>
__global__ void wgrad_thin_cin_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ partial,
                                      ThinParams p) {
  constexpr int M4 = (M + 3) / 4 * 4;       // rows are read back as float4 broadcasts: 4x fewer LDS than FMAs
  __shared__ __align__(16) float xs[THIN_PB][M4];
  const cgan_conv_desc& d = p.d;
  const int co = blockIdx.y * blockDim.x + threadIdx.x;
  const long long p0 = (long long)blockIdx.x * p.pix_per_block;
  const long long p1 = min(p.npix, p0 + p.pix_per_block);
  float acc[M];
#pragma unroll
  for (int m = 0; m < M; ++m) acc[m] = 0.f;
  for (long long pb = p0; pb < p1; pb += THIN_PB) {
    const int nb = (int)min((long long)THIN_PB, p1 - pb);
    __syncthreads();
    for (int e = threadIdx.x; e < nb * M4; e += blockDim.x) {
      int pi = e / M4, m = e % M4;
      int n, oh, ow;
      thin_pixel(pb + pi, d, n, oh, ow);
      int ci = m % d.cin, tap = m / d.cin;
      long long off = m < M ? thin_in_offset(p, n, oh, ow, tap / d.kw, tap % d.kw) : -1;
      xs[pi][m] = off < 0 ? 0.f : x[off + ci];
    }
    __syncthreads();
    if (co < d.cout) {
      for (int pi = 0; pi < nb; ++pi) {
        float g = dy[(pb + pi) * d.cout + co];
        float xv[M4];
#pragma unroll
        for (int m = 0; m < M4; m += 4) *reinterpret_cast<float4*>(&xv[m]) = *reinterpret_cast<const float4*>(&xs[pi][m]);
#pragma unroll
        for (int m = 0; m < M; ++m) acc[m] = fmaf(xv[m], g, acc[m]);
      }
    }
  }
  if (co < d.cout) {
#pragma unroll
    for (int m = 0; m < M; ++m) partial[((long long)blockIdx.x * M + m) * d.cout + co] = acc[m];
  }
}

// Cout <= 4: thread = input channel; acc[tap][co]
template <int TAPS, int CO>
__global__ void wgrad_thin_cout_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ partial,
                                       ThinParams p) {
  __shared__ float gs[THIN_PB][CO];
  __shared__ long long offs[THIN_PB][TAPS];
  const cgan_conv_desc& d = p.d;
  const int ci = blockIdx.y * blockDim.x + threadIdx.x;
  const long long p0 = (long long)blockIdx.x * p.pix_per_block;
  const long long p1 = min(p.npix, p0 + p.pix_per_block);
  float acc[TAPS][CO];
#pragma unroll
  for (int t = 0; t < TAPS; ++t)
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[t][c] = 0.f;
  for (long long pb = p0; pb < p1; pb += THIN_PB) {
    const int nb = (int)min((long long)THIN_PB, p1 - pb);
    __syncthreads();
    for (int e = threadIdx.x; e < nb * TAPS; e += blockDim.x) {
      int pi = e / TAPS, tap = e % TAPS;
      int n, oh, ow;
      thin_pixel(pb + pi, d, n, oh, ow);
      offs[pi][tap] = thin_in_offset(p, n, oh, ow, tap / d.kw, tap % d.kw);
    }
    for (int e = threadIdx.x; e < nb * CO; e += blockDim.x) gs[e / CO][e % CO] = dy[(pb + e / CO) * d.cout + e % CO];
    __syncthreads();
    if (ci < d.cin) {
      for (int pi = 0; pi < nb; ++pi) {
        float g[CO];
#pragma unroll
        for (int c = 0; c < CO; ++c) g[c] = gs[pi][c];
#pragma unroll
        for (int t = 0; t < TAPS; ++t) {
          long long off = offs[pi][t];
          float xv = off < 0 ? 0.f : x[off + ci];
#pragma unroll
          for (int c = 0; c < CO; ++c) acc[t][c] = fmaf(xv, g[c], acc[t][c]);
        }
      }
    }
  }
  if (ci < d.cin) {
#pragma unroll
    for (int t = 0; t < TAPS; ++t)
#pragma unroll
      for (int c = 0; c < CO; ++c)
        partial[(((long long)blockIdx.x * TAPS + t) * d.cin + ci) * CO + c] = acc[t][c];
  }
}

// Forward of the same image-side layers (3 input channels: the first conv of every discriminator and of Inception):
// 27 x Cout per pixel is far below a tensor-core tile, so thread = output channel with the filter column in registers,
// the receptive fields of THIN_PB pixels staged in smem and read back as float4 broadcasts; stores are 128-byte rows.
template <int M4>
__global__ void fwd_thin_cin_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                    float* __restrict__ y, ThinParams p, int m_real, int relu, int ldy) {
  __shared__ __align__(16) float xs[THIN_PB][M4];
  const cgan_conv_desc& d = p.d;
  const int co = blockIdx.y * blockDim.x + threadIdx.x;
  const bool co_ok = co < d.cout;
  float wr[M4];
#pragma unroll
  for (int m = 0; m < M4; ++m) wr[m] = (co_ok && m < m_real) ? w[(long long)m * d.cout + co] : 0.f;
  const float b = (co_ok && bias) ? bias[co] : 0.f;
  const long long p0 = (long long)blockIdx.x * p.pix_per_block;
  const long long p1 = min(p.npix, p0 + p.pix_per_block);
  for (long long pb = p0; pb < p1; pb += THIN_PB) {
    const int nb = (int)min((long long)THIN_PB, p1 - pb);
    __syncthreads();
    for (int e = threadIdx.x; e < nb * M4; e += blockDim.x) {
      int pi = e / M4, m = e % M4;
      int n, oh, ow;
      thin_pixel(pb + pi, d, n, oh, ow);
      int ci = m % d.cin, tap = m / d.cin;
      long long off = m < m_real ? thin_in_offset(p, n, oh, ow, tap / d.kw, tap % d.kw) : -1;
      xs[pi][m] = off < 0 ? 0.f : x[off + ci];
    }
    __syncthreads();
    if (co_ok) {
      for (int pi = 0; pi < nb; ++pi) {
        float xv[M4];
#pragma unroll
        for (int m = 0; m < M4; m += 4) *reinterpret_cast<float4*>(&xv[m]) = *reinterpret_cast<const float4*>(&xs[pi][m]);
        float acc = 0.f;
#pragma unroll
        for (int m = 0; m < M4; ++m) acc = fmaf(xv[m], wr[m], acc);
        acc += b;
        if (relu) acc = fmaxf(acc, 0.f);
        y[(pb + pi) * ldy + co] = acc;
      }
    }
  }
}

// ---- 3x3 kernels over <= 4 input channels, fast staging ------------------------------------------------------------
// The two kernels above spend most of their time computing addresses in the staging loop (a pixel decode with two
// divisions per ELEMENT).  Here a CTA walks chunks of up to THIN_PB consecutive output pixels of ONE output row, so the
// chunk origin (image, row, first column) is decoded once per chunk and every per-element quantity (tap, channel, kh, kw)
// comes from compile-time divisors; all index arithmetic is 32-bit.
template <int CIN>
struct Thin3 {
  static constexpr int M = 9 * CIN;
  static constexpr int M4 = (M + 3) / 4 * 4;
};

struct Thin3Params {
  int n, h, w, cout, stride, upsample, oh, ow, pad_t, pad_l;
  int vh, vw;                 // virtual (zero-inserted) input extent
  int chunks_per_row;         // ceil(ow / THIN_PB)
  int nchunks;                // n * oh * chunks_per_row
  int chunks_per_block;
  int ld;                     // pixel stride of the output (fwd) in floats
};

// stage the receptive fields of `nb` pixels (row `oh` of image `img`, columns ow0..) as [pixel][M4] records
template <int CIN>
__device__ __forceinline__ void thin3_stage(float (*xs)[Thin3<CIN>::M4], const float* __restrict__ x, const Thin3Params& p,
                                            int img, int oh, int ow0, int nb) {
  constexpr int M = Thin3<CIN>::M, M4 = Thin3<CIN>::M4;
  const int row_base = img * p.h;
  for (int e = threadIdx.x; e < nb * M4; e += blockDim.x) {
    const int pi = e / M4, m = e - pi * M4;
    float v = 0.f;
    if (m < M) {
      const int tap = m / CIN, ci = m - tap * CIN;
      const int kh = tap / 3, kw = tap - kh * 3;
      int vh = oh * p.stride + kh - p.pad_t, vw = (ow0 + pi) * p.stride + kw - p.pad_l;
      bool ok = vh >= 0 && vw >= 0 && vh < p.vh && vw < p.vw;
      if (p.upsample) {
        ok = ok && !((vh | vw) & 1);
        vh >>= 1; vw >>= 1;
      }
      if (ok) v = __ldg(x + ((size_t)(row_base + vh) * p.w + vw) * CIN + ci);
    }
    xs[pi][m] = v;
  }
}

// (A variant with four output channels per thread — one LDS.128 feeding 16 FMAs — was measured in round 2: 160 registers per
// thread cut the occupancy to 3 CTAs per SM and it ran 20-35 % SLOWER than one channel per thread, which is bound by the
// FP32 pipe (27 FFMAs per pixel and channel = ~100 us for 512x32x32x128 outputs) plus the staging phases.)
template <int CIN>
__global__ void __launch_bounds__(128, 8)
fwd_thin3_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias, float* __restrict__ y,
                 const Thin3Params p, int relu, int round_out) {
  constexpr int M = Thin3<CIN>::M, M4 = Thin3<CIN>::M4;
  __shared__ __align__(16) float xs[THIN_PB][M4];
  const int co = blockIdx.y * blockDim.x + threadIdx.x;
  const bool co_ok = co < p.cout;
  float wr[M4];
#pragma unroll
  for (int m = 0; m < M4; ++m) wr[m] = (co_ok && m < M) ? w[(size_t)m * p.cout + co] : 0.f;
  const float b = (co_ok && bias) ? bias[co] : 0.f;
  const int c0 = blockIdx.x * p.chunks_per_block, c1 = min(p.nchunks, c0 + p.chunks_per_block);
  for (int c = c0; c < c1; ++c) {
    const int rowid = c / p.chunks_per_row, ow0 = (c - rowid * p.chunks_per_row) * THIN_PB;
    const int img = rowid / p.oh, oh = rowid - img * p.oh;
    const int nb = min(THIN_PB, p.ow - ow0);
    __syncthreads();
    thin3_stage<CIN>(xs, x, p, img, oh, ow0, nb);
    __syncthreads();
    if (co_ok) {
      float* yrow = y + ((size_t)rowid * p.ow + ow0) * p.ld + co;
#pragma unroll 2
      for (int pi = 0; pi < nb; ++pi) {
        float xv[M4];
#pragma unroll
        for (int m = 0; m < M4; m += 4) *reinterpret_cast<float4*>(&xv[m]) = *reinterpret_cast<const float4*>(&xs[pi][m]);
        float acc = b;
#pragma unroll
        for (int m = 0; m < M; ++m) acc = fmaf(xv[m], wr[m], acc);
        if (relu) acc = fmaxf(acc, 0.f);
        if (round_out) acc = rna_tf32(acc);  // the consumer is a tensor-core convolution: store TF32-representable values
        yrow[(size_t)pi * p.ld] = acc;
      }
    }
  }
}

// dW partial per CTA: thread = output channel, acc[m] over m = (tap, ci); dY is read exactly once, in 128-byte rows
template <int CIN>
__global__ void __launch_bounds__(128, 6)
wgrad_thin3_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ partial, const Thin3Params p) {
  constexpr int M = Thin3<CIN>::M, M4 = Thin3<CIN>::M4;
  __shared__ __align__(16) float xs[THIN_PB][M4];
  const int co = blockIdx.y * blockDim.x + threadIdx.x;
  const bool co_ok = co < p.cout;
  float acc[M];
#pragma unroll
  for (int m = 0; m < M; ++m) acc[m] = 0.f;
  const int c0 = blockIdx.x * p.chunks_per_block, c1 = min(p.nchunks, c0 + p.chunks_per_block);
  for (int c = c0; c < c1; ++c) {
    const int rowid = c / p.chunks_per_row, ow0 = (c - rowid * p.chunks_per_row) * THIN_PB;
    const int img = rowid / p.oh, oh = rowid - img * p.oh;
    const int nb = min(THIN_PB, p.ow - ow0);
    __syncthreads();
    thin3_stage<CIN>(xs, x, p, img, oh, ow0, nb);
    __syncthreads();
    if (co_ok) {
      const float* grow = dy + ((size_t)rowid * p.ow + ow0) * p.cout + co;
#pragma unroll 2
      for (int pi = 0; pi < nb; ++pi) {
        const float g = __ldg(grow + (size_t)pi * p.cout);
        float xv[M4];
#pragma unroll
        for (int m = 0; m < M4; m += 4) *reinterpret_cast<float4*>(&xv[m]) = *reinterpret_cast<const float4*>(&xs[pi][m]);
#pragma unroll
        for (int m = 0; m < M; ++m) acc[m] = fmaf(xv[m], g, acc[m]);
      }
    }
  }
  if (co_ok) {
#pragma unroll
    for (int m = 0; m < M; ++m) partial[((size_t)blockIdx.x * M + m) * p.cout + co] = acc[m];
  }
}

inline bool thin3_params(const cgan_conv_desc* d, int num_sms, int ctas_per_sm, int co_blocks, Thin3Params* p) {
  if (d->kh != 3 || d->kw != 3 || d->cin < 1 || d->cin > 4) return false;
  p->n = d->n; p->h = d->h; p->w = d->w; p->cout = d->cout; p->stride = d->stride; p->upsample = d->upsample;
  p->oh = d->oh; p->ow = d->ow; p->pad_t = d->pad_t; p->pad_l = d->pad_l;
  p->vh = d->upsample ? 2 * d->h : d->h;
  p->vw = d->upsample ? 2 * d->w : d->w;
  p->chunks_per_row = (d->ow + THIN_PB - 1) / THIN_PB;
  long long nchunks = (long long)d->n * d->oh * p->chunks_per_row;
  if (nchunks >= (1ll << 30) || (long long)d->n * d->h * d->w * d->cin >= (1ll << 31)) return false;
  p->nchunks = (int)nchunks;
  long long want = (long long)num_sms * ctas_per_sm / (co_blocks > 0 ? co_blocks : 1);
  if (want < 1) want = 1;
  p->chunks_per_block = (int)((nchunks + want - 1) / want);
  if (p->chunks_per_block < 1) p->chunks_per_block = 1;
  p->ld = d->cout;
  return true;
}

}  // namespace

// ---- 1x1 kernels over <= 4 input channels (the shortcut of BigGAN's first discriminator block, resnet_biggan.py:
// a 3 -> ch pointwise conv at full image resolution) ----------------------------------------------------------------------
// Both are streams over the [pixels, cout] tensor: the forward writes it once (thread = 4 output channels of one pixel,
// filter rows in registers; residual add, ReLU and TF32 rounding fused), the filter gradient reads it once (thread =
// output channel, PWT_U pixels in flight, one partial [cin, cout] per CTA).
template <int CIN>
__global__ void fwd_pw_thin_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                   float* __restrict__ y, const float* __restrict__ residual, long long npix, int cout,
                                   int ldy, int relu, int round_out) {
  const int q = cout >> 2;                                   // float4 columns per pixel
  const long long total = npix * q;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long pix = e / q;
    const int c = (int)(e - pix * q) * 4;
    float4 acc = bias ? __ldg(reinterpret_cast<const float4*>(bias + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int ci = 0; ci < CIN; ++ci) {
      const float xv = __ldg(x + pix * CIN + ci);
      const float4 wv = __ldg(reinterpret_cast<const float4*>(w + (long long)ci * cout + c));
      acc.x = fmaf(xv, wv.x, acc.x); acc.y = fmaf(xv, wv.y, acc.y); acc.z = fmaf(xv, wv.z, acc.z); acc.w = fmaf(xv, wv.w, acc.w);
    }
    const long long o = pix * ldy + c;
    if (residual) {
      const float4 r = *reinterpret_cast<const float4*>(residual + o);
      acc.x += r.x; acc.y += r.y; acc.z += r.z; acc.w += r.w;
    }
    if (relu) { acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f); }
    if (round_out) { acc.x = rna_tf32(acc.x); acc.y = rna_tf32(acc.y); acc.z = rna_tf32(acc.z); acc.w = rna_tf32(acc.w); }
    *reinterpret_cast<float4*>(y + o) = acc;
  }
}

constexpr int PWT_U = 8;
template <int CIN>
__global__ void __launch_bounds__(128)
wgrad_pw_thin_kernel(const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ partial, long long npix,
                     int cout, long long pix_per_block) {
  const int co = blockIdx.y * blockDim.x + threadIdx.x;
  const bool co_ok = co < cout;
  float acc[CIN];
#pragma unroll
  for (int ci = 0; ci < CIN; ++ci) acc[ci] = 0.f;
  const long long p0 = (long long)blockIdx.x * pix_per_block, p1 = min(npix, p0 + pix_per_block);
  if (co_ok) {
    long long pix = p0;
    for (; pix + PWT_U <= p1; pix += PWT_U) {
      float g[PWT_U];
#pragma unroll
      for (int u = 0; u < PWT_U; ++u) g[u] = __ldg(dy + (pix + u) * cout + co);
#pragma unroll
      for (int u = 0; u < PWT_U; ++u)
#pragma unroll
        for (int ci = 0; ci < CIN; ++ci) acc[ci] = fmaf(__ldg(x + (pix + u) * CIN + ci), g[u], acc[ci]);
    }
    for (; pix < p1; ++pix) {
      const float g = __ldg(dy + pix * cout + co);
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) acc[ci] = fmaf(__ldg(x + pix * CIN + ci), g, acc[ci]);
    }
#pragma unroll
    for (int ci = 0; ci < CIN; ++ci) partial[((size_t)blockIdx.x * CIN + ci) * cout + co] = acc[ci];
  }
}

bool cgan_pw_thin_ok(const cgan_conv_desc* d) {       // 1x1, stride 1, <= 4 input channels: the pointwise stream kernels
  return d->kh == 1 && d->kw == 1 && d->stride == 1 && !d->upsample && d->cin >= 1 && d->cin <= 4 && d->cout >= 16 &&
         d->cout % 4 == 0 && d->oh == d->h && d->ow == d->w;
}

int cgan_fwd_pw_thin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, float* y,
                     const float* residual, int relu, int ldy, int round_out) {
  const long long npix = (long long)d->n * d->h * d->w;
  if (npix == 0) return CGAN_OK;
  const long long total = npix * (d->cout / 4);
  long long blocks = (total + 255) / 256;
  const long long cap = 16ll * ctx->num_sms;
  if (blocks > cap) blocks = cap;
  switch (d->cin) {
    case 1: fwd_pw_thin_kernel<1><<<(unsigned)blocks, 256, 0, ctx->stream>>>(x, w, bias, y, residual, npix, d->cout, ldy, relu, round_out); break;
    case 2: fwd_pw_thin_kernel<2><<<(unsigned)blocks, 256, 0, ctx->stream>>>(x, w, bias, y, residual, npix, d->cout, ldy, relu, round_out); break;
    case 3: fwd_pw_thin_kernel<3><<<(unsigned)blocks, 256, 0, ctx->stream>>>(x, w, bias, y, residual, npix, d->cout, ldy, relu, round_out); break;
    default: fwd_pw_thin_kernel<4><<<(unsigned)blocks, 256, 0, ctx->stream>>>(x, w, bias, y, residual, npix, d->cout, ldy, relu, round_out); break;
  }
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

bool cgan_wgrad_thin_ok(const cgan_conv_desc* d) {
  if ((long long)d->n * d->oh * d->ow >= (1ll << 31)) return false;      // 32-bit pixel arithmetic in the kernels
  int m = d->kh * d->kw * d->cin;
  if (cgan_pw_thin_ok(d)) return true;
  if (d->cin <= 4 && (m == 9 || m == 18 || m == 27 || m == 36) && d->kh == 3 && d->kw == 3) return true;
  if (d->cout <= 4 && d->cout == 3 && d->kh == 3 && d->kw == 3) return true;
  return false;
}

int cgan_wgrad_thin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, float* dw) {
  ThinParams p;
  p.d = *d;
  p.vh = d->upsample ? 2 * d->h : d->h;
  p.vw = d->upsample ? 2 * d->w : d->w;
  p.npix = (long long)d->n * d->oh * d->ow;
  if (p.npix >= (1ll << 31)) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: more than 2^31 output pixels%s", "cgan_wgrad_thin");
  if (cgan_pw_thin_ok(d)) {
    const int co_blocks = (d->cout + 127) / 128;
    long long want = 8ll * ctx->num_sms / co_blocks;
    long long ppb = (p.npix + want - 1) / want;
    ppb = (ppb + PWT_U - 1) / PWT_U * PWT_U;
    const int blocks = (int)((p.npix + ppb - 1) / ppb);
    const long long wn = (long long)d->cin * d->cout;
    void* ws = nullptr;
    int rc = cgan_ws(ctx, (size_t)blocks * wn * sizeof(float), &ws);
    if (rc) return rc;
    float* partial = reinterpret_cast<float*>(ws);
    dim3 grid(blocks, co_blocks);
    switch (d->cin) {
      case 1: wgrad_pw_thin_kernel<1><<<grid, 128, 0, ctx->stream>>>(x, dy, partial, p.npix, d->cout, ppb); break;
      case 2: wgrad_pw_thin_kernel<2><<<grid, 128, 0, ctx->stream>>>(x, dy, partial, p.npix, d->cout, ppb); break;
      case 3: wgrad_pw_thin_kernel<3><<<grid, 128, 0, ctx->stream>>>(x, dy, partial, p.npix, d->cout, ppb); break;
      default: wgrad_pw_thin_kernel<4><<<grid, 128, 0, ctx->stream>>>(x, dy, partial, p.npix, d->cout, ppb); break;
    }
    CGAN_LAUNCHED(ctx);
    return cgan_splitk_reduce(ctx, dw, partial, wn, blocks);
  }
  if (d->cin <= 4 && d->kh == 3 && d->kw == 3) {
    Thin3Params q;
    const int co_blocks = (d->cout + 127) / 128;
    if (thin3_params(d, ctx->num_sms, 6, co_blocks, &q)) {
      const int blocks = (q.nchunks + q.chunks_per_block - 1) / q.chunks_per_block;
      const long long wn = 9ll * d->cin * d->cout;
      void* ws = nullptr;
      int rc = cgan_ws(ctx, (size_t)blocks * wn * sizeof(float), &ws);
      if (rc) return rc;
      float* partial = reinterpret_cast<float*>(ws);
      dim3 grid(blocks, co_blocks);
      switch (d->cin) {
        case 1: wgrad_thin3_kernel<1><<<grid, 128, 0, ctx->stream>>>(x, dy, partial, q); break;
        case 2: wgrad_thin3_kernel<2><<<grid, 128, 0, ctx->stream>>>(x, dy, partial, q); break;
        case 3: wgrad_thin3_kernel<3><<<grid, 128, 0, ctx->stream>>>(x, dy, partial, q); break;
        default: wgrad_thin3_kernel<4><<<grid, 128, 0, ctx->stream>>>(x, dy, partial, q); break;
      }
      CGAN_LAUNCHED(ctx);
      return cgan_splitk_reduce(ctx, dw, partial, wn, blocks);
    }
  }
  long long want_blocks = 4ll * ctx->num_sms;
  long long ppb = (p.npix + want_blocks - 1) / want_blocks;
  ppb = (ppb + THIN_PB - 1) / THIN_PB * THIN_PB;
  p.pix_per_block = ppb;
  int blocks = (int)((p.npix + ppb - 1) / ppb);
  long long wn = (long long)d->kh * d->kw * d->cin * d->cout;
  void* ws = nullptr;
  int rc = cgan_ws(ctx, (size_t)blocks * wn * sizeof(float), &ws);
  if (rc) return rc;
  float* partial = reinterpret_cast<float*>(ws);
  if (d->cin <= 4) {
    int threads = d->cout >= 256 ? 256 : ((d->cout + 31) / 32 * 32);
    dim3 grid(blocks, (d->cout + threads - 1) / threads);
    int m = d->kh * d->kw * d->cin;
    if (m == 9) wgrad_thin_cin_kernel<9><<<grid, threads, 0, ctx->stream>>>(x, dy, partial, p);
    else if (m == 18) wgrad_thin_cin_kernel<18><<<grid, threads, 0, ctx->stream>>>(x, dy, partial, p);
    else if (m == 27) wgrad_thin_cin_kernel<27><<<grid, threads, 0, ctx->stream>>>(x, dy, partial, p);
    else wgrad_thin_cin_kernel<36><<<grid, threads, 0, ctx->stream>>>(x, dy, partial, p);
  } else {
    int threads = d->cin >= 256 ? 256 : ((d->cin + 31) / 32 * 32);
    dim3 grid(blocks, (d->cin + threads - 1) / threads);
    wgrad_thin_cout_kernel<9, 3><<<grid, threads, 0, ctx->stream>>>(x, dy, partial, p);
  }
  CGAN_LAUNCHED(ctx);
  return cgan_splitk_reduce(ctx, dw, partial, wn, blocks);
}


bool cgan_fwd_thin_ok(const cgan_conv_desc* d) {
  if ((long long)d->n * d->oh * d->ow >= (1ll << 31)) return false;
  return d->cin <= 4 && d->kh * d->kw * d->cin <= THIN_MAX_M && d->cout >= 16;
}

bool cgan_fwd_thin3_ok(const cgan_conv_desc* d) {      // the fast 3x3 kernel (which also fuses ReLU + TF32 rounding) applies
  Thin3Params q;
  return cgan_fwd_thin_ok(d) && d->kh == 3 && d->kw == 3 && thin3_params(d, 148, 6, 1, &q);
}

int cgan_fwd_thin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, float* y, int relu,
                  int ldy, int round_out) {
  ThinParams p;
  p.d = *d;
  p.vh = d->upsample ? 2 * d->h : d->h;
  p.vw = d->upsample ? 2 * d->w : d->w;
  p.npix = (long long)d->n * d->oh * d->ow;
  if (d->kh == 3 && d->kw == 3) {
    Thin3Params q;
    const int threads3 = d->cout >= 128 ? 128 : ((d->cout + 31) / 32 * 32);
    const int co_blocks3 = (d->cout + threads3 - 1) / threads3;
    if (thin3_params(d, ctx->num_sms, 8 * 128 / threads3, co_blocks3, &q)) {
      q.ld = ldy;
      dim3 grid((q.nchunks + q.chunks_per_block - 1) / q.chunks_per_block, co_blocks3);
      switch (d->cin) {
        case 1: fwd_thin3_kernel<1><<<grid, threads3, 0, ctx->stream>>>(x, w, bias, y, q, relu, round_out); break;
        case 2: fwd_thin3_kernel<2><<<grid, threads3, 0, ctx->stream>>>(x, w, bias, y, q, relu, round_out); break;
        case 3: fwd_thin3_kernel<3><<<grid, threads3, 0, ctx->stream>>>(x, w, bias, y, q, relu, round_out); break;
        default: fwd_thin3_kernel<4><<<grid, threads3, 0, ctx->stream>>>(x, w, bias, y, q, relu, round_out); break;
      }
      CGAN_LAUNCHED(ctx);
      return CGAN_OK;
    }
  }
  const int threads = d->cout >= 128 ? 128 : ((d->cout + 31) / 32 * 32);
  const int co_blocks = (d->cout + threads - 1) / threads;
  long long want_blocks = 16ll * ctx->num_sms * 128 / threads / co_blocks;     // ~16 resident warps' worth of CTAs per SM, x2 waves
  if (want_blocks < 1) want_blocks = 1;
  long long ppb = (p.npix + want_blocks - 1) / want_blocks;
  ppb = (ppb + THIN_PB - 1) / THIN_PB * THIN_PB;
  p.pix_per_block = ppb;
  dim3 grid((unsigned)((p.npix + ppb - 1) / ppb), (unsigned)co_blocks);
  const int m = d->kh * d->kw * d->cin;
  if (m <= 12) fwd_thin_cin_kernel<12><<<grid, threads, 0, ctx->stream>>>(x, w, bias, y, p, m, relu, ldy);
  else if (m <= 20) fwd_thin_cin_kernel<20><<<grid, threads, 0, ctx->stream>>>(x, w, bias, y, p, m, relu, ldy);
  else if (m <= 28) fwd_thin_cin_kernel<28><<<grid, threads, 0, ctx->stream>>>(x, w, bias, y, p, m, relu, ldy);
  else fwd_thin_cin_kernel<36><<<grid, threads, 0, ctx->stream>>>(x, w, bias, y, p, m, relu, ldy);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}
