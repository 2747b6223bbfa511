// Image-side ("thin") convolutions on the tensor cores — math_mode 1.
//
// The first convolution of every discriminator (3 input channels), the last of every generator (3 output channels) and
// Inception's stem are contractions over kh*kw*3 = 27 values per pixel: far too skinny for an implicit GEMM over
// 32-channel k-blocks (the tap loop would move the 256-channel operand nine times for 3 output channels) and, as fp32
// streaming kernels (thin.cu), bound by the FP32 pipe at several times their HBM time.
// Here each becomes ONE dense 32-wide GEMM on the existing wgmma kernels plus a streaming pass:
//
//   cin <= 4   forward   : P = patches(x) [pixels, 32]  ->  y  = P W            (1x1 wgmma conv, fused epilogue)
//              filter    : dW = P^T dy                                            (wgmma filter-gradient kernel)
//              input grad: T = dy W^T [pixels, 32]      ->  dx = shift_add(T)     (stride 1 or 2)
//   cout <= 4  forward   : T = x W' [pixels, 32]        ->  y  = shift_add(T) + bias
//              input grad: P = patches(dy)              ->  dx = P W'^T
//              filter    : dW' = x^T P                                            (then re-laid out to HWIO)
//
// patches() gathers the kh*kw*C <= 32 values a pixel's taps see into one 128-byte row (zero where SAME padding applies,
// TF32-rounded: the GEMM skips its operand rounding); shift_add() is its adjoint: out[p, c] = sum_tap T[p + off(tap), tap*C + c].
// Both stream a [pixels, 32] fp32 tensor once (1/4 of a 128-channel activation).  Arithmetic: TF32 operands, fp32
// accumulation — the same as every other tensor-core contraction of math_mode 1 (CGAN_PATH_TCGEN05_TF32).
#include "common.cuh"

namespace {

constexpr int TT_K = 32;                        // patch row: 32 floats = one 128-byte TMA / swizzle row
constexpr size_t TT_RESERVE = 16u << 20;        // head of the workspace left to the GEMM kernels (weight prep, split-K partials)
constexpr int TT_MAX_TAPS = 32;

struct TapList {
  int ntaps, c, k;                              // k = ntaps * c <= 32
  int off_h[TT_MAX_TAPS], off_w[TT_MAX_TAPS];
};

// out[(n, gy, gx)][m], m = tap*C + c  =  src[n, gy*stride + off_h[tap], gx*stride + off_w[tap], c]  (0 outside / m >= K).
// One thread per (pixel, 4 consecutive m): eight threads write one 128-byte row.  A thread keeps its quarter-row index for
// the whole grid-stride loop (the stride is a multiple of 8), so the (tap, channel) decode of its four values happens once;
// per pixel it costs one 32-bit decode, four predicated loads from the (L1 / L2 resident) 3-channel source and one STG.128.
__global__ void __launch_bounds__(256)
patch_kernel(float* __restrict__ out, const float* __restrict__ src, TapList t, int n, int gh, int gw, int sh, int sw, int stride) {
  const unsigned tid = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned q = tid & 7u;
  int dy[4], dx[4], cc[4];
  bool live[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int m = (int)q * 4 + j;
    live[j] = m < t.k;
    const int tap = live[j] ? m / t.c : 0;
    cc[j] = live[j] ? m - tap * t.c : 0;
    dy[j] = t.off_h[tap]; dx[j] = t.off_w[tap];
  }
  const unsigned npix = (unsigned)n * gh * gw;                // < 2^31 (host-checked)
  const unsigned pstep = (gridDim.x * blockDim.x) >> 3;
  for (unsigned pix = tid >> 3; pix < npix; pix += pstep) {
    const unsigned row = pix / (unsigned)gw;
    const int gx = (int)(pix - row * (unsigned)gw);
    const unsigned img = row / (unsigned)gh;
    const int gy = (int)(row - img * (unsigned)gh);
    const float* base = src + (size_t)img * sh * sw * t.c;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int y = gy * stride + dy[j], x = gx * stride + dx[j];
      const bool ok = live[j] && y >= 0 && y < sh && x >= 0 && x < sw;
      v[j] = ok ? rna_tf32(__ldg(base + ((size_t)y * sw + x) * t.c + cc[j])) : 0.f;
    }
    *reinterpret_cast<float4*>(out + (size_t)pix * TT_K + q * 4) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// out[(n, y, x)][c] = bias[c] + sum_tap T[(n, y + off_h[tap], x + off_w[tap])][tap*C + c]   (taps outside the th x tw grid: 0)
// STRIDE 2 (the input gradient of a stride-2 convolution): T row ((y + off_h) / 2, (x + off_w) / 2), only where both sums
// are even; an odd one is a tap that no output pixel of the forward convolution sends to (y, x)
template <int STRIDE>
__global__ void shift_add_kernel(float* __restrict__ out, const float* __restrict__ t32, const float* __restrict__ bias,
                                 TapList t, int n, int oh, int ow, int th, int tw, int relu) {
  const long long total = (long long)n * oh * ow;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    long long pix = i;
    const int x = (int)(pix % ow);
    pix /= ow;
    const int y = (int)(pix % oh);
    const int img = (int)(pix / oh);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (bias)
      for (int c = 0; c < t.c; ++c) acc[c] = bias[c];
    for (int tap = 0; tap < t.ntaps; ++tap) {
      int ty = y + t.off_h[tap], tx = x + t.off_w[tap];
      if (STRIDE == 2) {
        if ((ty | tx) & 1) continue;
        ty >>= 1; tx >>= 1;
      }
      if (ty < 0 || ty >= th || tx < 0 || tx >= tw) continue;
      const float* row = t32 + (((long long)img * th + ty) * tw + tx) * TT_K + tap * t.c;
      for (int c = 0; c < t.c; ++c) acc[c] += __ldg(row + c);
    }
    for (int c = 0; c < t.c; ++c) out[i * t.c + c] = relu ? fmaxf(acc[c], 0.f) : acc[c];
  }
}

// HWIO filter w[tap][ci][co] (co < C <= 4)  <->  W'[ci][ld] with W'[ci][tap*C + co]; columns >= ntaps*C are zero
__global__ void wcols_from_hwio_kernel(float* __restrict__ wp, const float* __restrict__ w, int ntaps, int cin, int c, int ld) {
  const int total = cin * ld;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int ci = i / ld, m = i - ci * ld;
    float v = 0.f;
    if (m < ntaps * c) {
      const int tap = m / c, co = m - tap * c;
      v = w[((long long)tap * cin + ci) * c + co];
    }
    wp[i] = v;
  }
}
// dst[rows_dst][cols] = src[rows_src][cols] followed by zero rows
__global__ void pad_rows_kernel(float* __restrict__ dst, const float* __restrict__ src, int rows_src, int rows_dst, int cols) {
  const int total = rows_dst * cols;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x)
    dst[i] = (i / cols) < rows_src ? src[i] : 0.f;
}
__global__ void hwio_from_wcols_kernel(float* __restrict__ w, const float* __restrict__ wp, int ntaps, int cin, int c, int ld) {
  const int total = ntaps * cin * c;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int co = i % c, ci = (i / c) % cin, tap = i / (c * cin);
    w[i] = wp[(long long)ci * ld + tap * c + co];
  }
}

inline int ew_blocks(cgan_ctx* ctx, long long n) {
  long long b = (n + 255) / 256, cap = (long long)ctx->num_sms * 32;
  return (int)(b < cap ? (b < 1 ? 1 : b) : cap);
}

// direct taps of the convolution d over C channels: sign +1, the forward taps (tap (kh, kw) reads the input at
// output*stride + (kh - pad_t, kw - pad_l)); -1, the adjoint taps (stride 1: input pixel ih receives tap kh from output row
// ih + pad_t - kh)
inline void tap_list(const cgan_conv_desc* d, int sign, int c, TapList* t) {
  ConvTaps ct;
  conv_taps(d, sign, TAP_DIRECT, &ct);
  t->ntaps = ct.ntaps; t->c = c; t->k = ct.ntaps * c;
  for (int i = 0; i < ct.ntaps; ++i) { t->off_h[i] = ct.off_h[i]; t->off_w[i] = ct.off_w[i]; }
}

// y = x W over a dense NHWC [n, h, w, kdim] operand: a 1x1 convolution on the tensor cores
inline TcConv tc_gemm(const float* x, int n, int h, int w, int kdim, const float* wsrc, int transpose_w, int ncols, float* y,
                      int ldy) {
  TcConv c = {};
  tc_in_dense(&c.a, x, n, h, w, kdim);
  c.wsrc = wsrc; c.taps_total = 1; c.transpose_w = transpose_w; c.ncols = ncols;
  c.taps.ntaps = 1;
  tc_out_dense(&c, y, h, w, ldy);
  return c;
}

// dw[xch][dych] = x^T dy over dense NHWC operands on an n x h x w grid: the filter gradient of a 1x1 convolution
inline TcWgrad tc_gemm_tn(int n, int h, int w, const float* x, int xch, int x_tf32, const float* dy, int dych, int dy_tf32,
                          float* dw) {
  TcWgrad g = {};
  tc_in_dense(&g.x, x, n, h, w, xch);
  tc_in_dense(&g.dy, dy, n, h, w, dych);
  g.x.tf32 = x_tf32; g.dy.tf32 = dy_tf32;
  g.taps.ntaps = 1; g.taps_total = 1; g.dw = dw;
  return g;
}

// workspace: [0, TT_RESERVE) for the GEMM kernels' own use | patch / T tensor | small weight buffers (2 x 64 KB)
inline int tt_workspace(cgan_ctx* ctx, long long pixels, float** big, float** small0, float** small1) {
  const size_t big_bytes = ((size_t)pixels * TT_K * sizeof(float) + 255) / 256 * 256;
  void* ws = nullptr;
  int rc = cgan_ws(ctx, TT_RESERVE + big_bytes + (128u << 10), &ws);
  if (rc) return rc;
  char* b = reinterpret_cast<char*>(ws) + TT_RESERVE;
  *big = reinterpret_cast<float*>(b);
  *small0 = reinterpret_cast<float*>(b + big_bytes);
  *small1 = reinterpret_cast<float*>(b + big_bytes + (64u << 10));
  return CGAN_OK;
}

inline bool common_ok(cgan_ctx* ctx, const cgan_conv_desc* d) {
  return ctx->math_mode == 1 && !d->upsample && d->kh * d->kw <= TT_MAX_TAPS && d->n >= 1 &&
         (long long)d->n * d->oh * d->ow < (1ll << 31) && (long long)d->n * d->h * d->w < (1ll << 31);
}
inline bool stride1_same_grid(const cgan_conv_desc* d) { return d->stride == 1 && d->oh == d->h && d->ow == d->w; }
inline bool stride2_same_grid(const cgan_conv_desc* d) {
  return d->stride == 2 && d->oh == (d->h + 1) / 2 && d->ow == (d->w + 1) / 2;
}

}  // namespace

// ---- cin <= 4 -------------------------------------------------------------------------------------------------------------
bool cgan_thin_tc_cin_ok(cgan_ctx* ctx, const cgan_conv_desc* d) {
  return common_ok(ctx, d) && d->cin >= 1 && d->cin <= 4 && d->kh * d->kw * d->cin <= TT_K && d->cout >= 16 && d->cout % 4 == 0 &&
         d->cout <= 512 && cgan_tc_shape_ok(d->n, d->oh, d->ow, TT_K, d->cout) &&
         (size_t)2 * ctx->num_sms * TT_K * d->cout * 4 <= TT_RESERVE;
}

int cgan_thin_tc_fwd_cin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const cgan_conv_epilogue* ep,
                         float* y) {
  const long long pixels = (long long)d->n * d->oh * d->ow;
  float *pt, *s0, *s1;
  int rc = tt_workspace(ctx, pixels, &pt, &s0, &s1);
  if (rc) return rc;
  TapList t;
  tap_list(d, 1, d->cin, &t);
  patch_kernel<<<ew_blocks(ctx, pixels * 8), 256, 0, ctx->stream>>>(pt, x, t, d->n, d->oh, d->ow, d->h, d->w, d->stride);
  CGAN_LAUNCHED(ctx);
  // HWIO flattened is [K = kh*kw*cin][cout]: padded to 32 rows so that the GEMM sees plain 32-channel operands
  pad_rows_kernel<<<cdiv((long long)TT_K * d->cout, 256), 256, 0, ctx->stream>>>(s0, w, t.k, TT_K, d->cout);
  CGAN_LAUNCHED(ctx);
  // y = P W: a 1x1 convolution over the 32-channel patch tensor
  TcConv c = tc_gemm(pt, d->n, d->oh, d->ow, TT_K, s0, 1, d->cout, y, (ep && ep->ldy) ? ep->ldy : d->cout);
  tc_set_epilogue(&c, ep, true);
  return cgan_conv_tc(ctx, c);
}

// The filter-gradient products below read the patch tensor and write into the workspace, whose slices are 256-byte
// aligned, and the caller checks the alignment of x and dy: their _ok tests describe them with null pointers.
bool cgan_thin_tc_wgrad_cin_ok(cgan_ctx* ctx, const cgan_conv_desc* d) {
  return cgan_thin_tc_cin_ok(ctx, d) && d->cout <= 256 &&
         cgan_wgrad_tc_fits(tc_gemm_tn(d->n, d->oh, d->ow, nullptr, TT_K, 1, nullptr, d->cout, 0, nullptr));
}

int cgan_thin_tc_wgrad_cin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, int dy_tf32, float* dw) {
  const long long pixels = (long long)d->n * d->oh * d->ow;
  float *pt, *s0, *s1;
  int rc = tt_workspace(ctx, pixels, &pt, &s0, &s1);
  if (rc) return rc;
  TapList t;
  tap_list(d, 1, d->cin, &t);
  patch_kernel<<<ew_blocks(ctx, pixels * 8), 256, 0, ctx->stream>>>(pt, x, t, d->n, d->oh, d->ow, d->h, d->w, d->stride);
  CGAN_LAUNCHED(ctx);
  // dW32[32][cout] = P^T dy over the output grid
  rc = cgan_wgrad_tc(ctx, tc_gemm_tn(d->n, d->oh, d->ow, pt, TT_K, 1, dy, d->cout, dy_tf32, s0));
  if (rc) return rc;
  return cgan_copy(ctx, dw, s0, (int64_t)t.k * d->cout);          // rows [0, K) of dW32 are HWIO's [kh][kw][cin][cout]
}

bool cgan_thin_tc_dgrad_cin_ok(cgan_ctx* ctx, const cgan_conv_desc* d) {
  return common_ok(ctx, d) && (stride1_same_grid(d) || stride2_same_grid(d)) && d->cin >= 1 && d->cin <= 4 &&
         d->kh * d->kw * d->cin <= TT_K && d->cout >= 8 &&
         d->cout % 4 == 0 && cgan_tc_shape_ok(d->n, d->oh, d->ow, d->cout, TT_K);
}

int cgan_thin_tc_dgrad_cin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* dy, const float* w, const cgan_conv_epilogue* ep,
                           float* dx) {
  const long long pixels = (long long)d->n * d->oh * d->ow;
  float *tt, *s0, *s1;
  int rc = tt_workspace(ctx, pixels, &tt, &s0, &s1);
  if (rc) return rc;
  TapList t;
  tap_list(d, -1, d->cin, &t);
  // T[p][tap*cin + ci] = sum_co dy[p][co] w[tap][ci][co]: HWIO flattened is [ncols = K][kdim = cout]
  TcConv c = tc_gemm(dy, d->n, d->oh, d->ow, d->cout, w, 0, t.k, tt, TT_K);
  tc_set_epilogue(&c, nullptr, ep && (ep->flags & CGAN_CONV_IN_TF32));
  rc = cgan_conv_tc(ctx, c);
  if (rc) return rc;
  // dx gathers T over dy's grid: at stride 2, pixel i receives tap kh from dy row (i + pad_t - kh) / 2 when that is whole
  const int blocks = ew_blocks(ctx, (long long)d->n * d->h * d->w);
  if (d->stride == 2)
    shift_add_kernel<2><<<blocks, 256, 0, ctx->stream>>>(dx, tt, ep ? ep->bias : nullptr, t, d->n, d->h, d->w, d->oh, d->ow, 0);
  else
    shift_add_kernel<1><<<blocks, 256, 0, ctx->stream>>>(dx, tt, ep ? ep->bias : nullptr, t, d->n, d->h, d->w, d->oh, d->ow, 0);
  CGAN_LAUNCHED(ctx);
  if (ep_needs_post(ep, false))
    return cgan_conv_post_epilogue(ctx, dx, (int64_t)d->n * d->h * d->w, d->cin, d->cin, ep->residual, ep->mask, ep->mask_leak,
                                   (ep->flags & CGAN_CONV_RELU) ? 1 : 0, (ep->flags & CGAN_CONV_ROUND_OUT) ? 1 : 0);
  return CGAN_OK;
}

// ---- cout <= 4 ------------------------------------------------------------------------------------------------------------
bool cgan_thin_tc_cout_ok(cgan_ctx* ctx, const cgan_conv_desc* d) {
  return common_ok(ctx, d) && stride1_same_grid(d) && d->cout >= 1 && d->cout <= 4 && d->kh * d->kw * d->cout <= TT_K &&
         d->cin >= 32 && d->cin % 4 == 0 && d->cin <= 512 && cgan_tc_shape_ok(d->n, d->h, d->w, d->cin, TT_K);
}

int cgan_thin_tc_fwd_cout(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const cgan_conv_epilogue* ep,
                          float* y) {
  const long long pixels = (long long)d->n * d->h * d->w;
  float *tt, *wp, *s1;
  int rc = tt_workspace(ctx, pixels, &tt, &wp, &s1);
  if (rc) return rc;
  TapList t;
  tap_list(d, 1, d->cout, &t);
  wcols_from_hwio_kernel<<<cdiv((long long)d->cin * TT_K, 256), 256, 0, ctx->stream>>>(wp, w, t.ntaps, d->cin, d->cout, TT_K);
  CGAN_LAUNCHED(ctx);
  // T[p][tap*cout + co] = sum_ci x[p][ci] w[tap][ci][co]: every tap's contribution at the INPUT pixel, all taps in one GEMM
  TcConv c = tc_gemm(x, d->n, d->h, d->w, d->cin, wp, 1, TT_K, tt, TT_K);
  tc_set_epilogue(&c, nullptr, ep && (ep->flags & CGAN_CONV_IN_TF32));
  rc = cgan_conv_tc(ctx, c);
  if (rc) return rc;
  const bool post = ep_needs_post(ep, true);
  const int relu = (ep && (ep->flags & CGAN_CONV_RELU)) ? 1 : 0;
  shift_add_kernel<1><<<ew_blocks(ctx, pixels), 256, 0, ctx->stream>>>(y, tt, ep ? ep->bias : nullptr, t, d->n, d->oh, d->ow, d->h, d->w,
                                                                   post ? 0 : relu);
  CGAN_LAUNCHED(ctx);
  if (post)
    return cgan_conv_post_epilogue(ctx, y, (int64_t)pixels, d->cout, d->cout, ep->residual, ep->mask, ep->mask_leak, relu,
                                   (ep->flags & CGAN_CONV_ROUND_OUT) ? 1 : 0);
  return CGAN_OK;
}

int cgan_thin_tc_dgrad_cout(cgan_ctx* ctx, const cgan_conv_desc* d, const float* dy, const float* w, const cgan_conv_epilogue* ep,
                            float* dx) {
  const long long pixels = (long long)d->n * d->h * d->w;
  float *pt, *wp, *s1;
  int rc = tt_workspace(ctx, pixels, &pt, &wp, &s1);
  if (rc) return rc;
  TapList t;
  tap_list(d, -1, d->cout, &t);
  patch_kernel<<<ew_blocks(ctx, pixels * 8), 256, 0, ctx->stream>>>(pt, dy, t, d->n, d->h, d->w, d->oh, d->ow, 1);
  CGAN_LAUNCHED(ctx);
  wcols_from_hwio_kernel<<<cdiv((long long)d->cin * TT_K, 256), 256, 0, ctx->stream>>>(wp, w, t.ntaps, d->cin, d->cout, TT_K);
  CGAN_LAUNCHED(ctx);
  // dx[p][ci] = sum_m P[p][m] W'[ci][m]: W' [ncols = cin][kdim = 32], columns >= K zero
  TcConv c = tc_gemm(pt, d->n, d->h, d->w, TT_K, wp, 0, d->cin, dx, d->cin);
  tc_set_epilogue(&c, ep, true);
  return cgan_conv_tc(ctx, c);
}

bool cgan_thin_tc_wgrad_cout_ok(cgan_ctx* ctx, const cgan_conv_desc* d) {
  return cgan_thin_tc_cout_ok(ctx, d) && d->cin >= 64 &&
         cgan_wgrad_tc_fits(tc_gemm_tn(d->n, d->h, d->w, nullptr, d->cin, 0, nullptr, TT_K, 1, nullptr)) &&
         (size_t)2 * ctx->num_sms * TT_K * d->cin * 4 <= TT_RESERVE && (size_t)d->cin * TT_K * 4 <= (64u << 10);
}

int cgan_thin_tc_wgrad_cout(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, int x_tf32, float* dw) {
  const long long pixels = (long long)d->n * d->h * d->w;
  float *pt, *s0, *dwp;
  int rc = tt_workspace(ctx, pixels, &pt, &s0, &dwp);
  if (rc) return rc;
  TapList t;
  tap_list(d, -1, d->cout, &t);
  patch_kernel<<<ew_blocks(ctx, pixels * 8), 256, 0, ctx->stream>>>(pt, dy, t, d->n, d->h, d->w, d->oh, d->ow, 1);
  CGAN_LAUNCHED(ctx);
  // dW'[cin][32] = x^T P
  rc = cgan_wgrad_tc(ctx, tc_gemm_tn(d->n, d->h, d->w, x, d->cin, x_tf32, pt, TT_K, 1, dwp));
  if (rc) return rc;
  hwio_from_wcols_kernel<<<cdiv((long long)t.k * d->cin, 256), 256, 0, ctx->stream>>>(dw, dwp, t.ntaps, d->cin, d->cout, TT_K);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}
