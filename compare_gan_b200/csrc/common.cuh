// Shared helpers for the sm_90a kernels behind include/cgan_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/cgan_b200.h"

struct cgan_ctx {
  int device;
  cudaStream_t stream;
  void* ws;
  size_t ws_bytes;
  int math_mode;
  int64_t launches;
  int num_sms;
  int tc_mt_max;       // tensor-core kernels: max tiles per CTA sharing one operand tile (CGAN_OPT_TC_MT / env CGAN_TC_MT, default 2)
  int tc_halo;         // 3x3 stride-1 tensor-core convolutions use the halo variant (CGAN_OPT_TC_HALO / env CGAN_TC_HALO, default 1)
  int tc_thin;         // image-side (<= 4 channel) convolutions through 32-wide patch tensors on wgmma (CGAN_OPT_TC_THIN / env CGAN_TC_THIN)
  int last_path;       // CGAN_PATH_* of the most recent contraction (cgan_ctx_get_option(CGAN_OPT_LAST_PATH))
  int last_tc_bn, last_tc_mt, last_tc_halo;   // geometry of the most recent conv_tc launch (CGAN_OPT_LAST_TC_*)
  int last_tc_ctas_per_sm;                    // CTAs of that launch that fit on one SM (CGAN_OPT_LAST_TC_CTAS_PER_SM)
  int last_tc_ep_smem;                        // that launch prefetched its residual / mask (CGAN_OPT_LAST_TC_EP_SMEM)
  int last_tc_tma_store;                      // that launch stored its tiles by TMA (CGAN_OPT_LAST_TC_TMA_STORE)
  unsigned* counters;  // CGAN_NUM_COUNTERS zero-initialised tickets for single-launch two-stage reductions (norm.cu)
  void* p2p;           // peer-memory all-reduce state (p2p.cu), null until cgan_p2p_local_handle
  char err[512];
};

constexpr int CGAN_NUM_COUNTERS = 1 << 18;

static inline int cgan_fail(cgan_ctx* ctx, int code, const char* fmt, const char* a = "", const char* b = "") {
  if (ctx) snprintf(ctx->err, sizeof(ctx->err), fmt, a, b);
  return code;
}

#define CGAN_REQUIRE(ctx, cond, msg)                                              \
  do {                                                                            \
    if (!(cond)) return cgan_fail((ctx), CGAN_ERR_ARG, "%s: %s", __func__, msg);  \
  } while (0)

#define CGAN_CUDA(ctx, call)                                                                        \
  do {                                                                                              \
    cudaError_t e__ = (call);                                                                       \
    if (e__ != cudaSuccess) return cgan_fail((ctx), CGAN_ERR_CUDA, "%s: %s", __func__, cudaGetErrorString(e__)); \
  } while (0)

// after every kernel launch: count it and surface launch-configuration errors without synchronising
#define CGAN_LAUNCHED(ctx)                                                                          \
  do {                                                                                              \
    (ctx)->launches++;                                                                              \
    cudaError_t e__ = cudaGetLastError();                                                           \
    if (e__ != cudaSuccess) return cgan_fail((ctx), CGAN_ERR_CUDA, "%s: launch: %s", __func__, cudaGetErrorString(e__)); \
  } while (0)

// Workspace owned by the context; grows on demand outside stream capture only.
static inline int cgan_ws(cgan_ctx* ctx, size_t bytes, void** out) {
  if (bytes > ctx->ws_bytes) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(ctx->stream, &st);
    if (st != cudaStreamCaptureStatusNone)
      return cgan_fail(ctx, CGAN_ERR_WORKSPACE, "%s: workspace would grow during stream capture (warm up first)%s", "cgan_ws");
    size_t want = bytes + bytes / 4 + (1 << 20);
    want = (want + 255) / 256 * 256;
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess && ctx->ws) e = cudaFree(ctx->ws);
    ctx->ws = nullptr;
    ctx->ws_bytes = 0;
    if (e == cudaSuccess) e = cudaMalloc(&ctx->ws, want);
    if (e != cudaSuccess) return cgan_fail(ctx, CGAN_ERR_CUDA, "%s: %s", "cgan_ws", cudaGetErrorString(e));
    ctx->ws_bytes = want;
  }
  *out = ctx->ws;
  return CGAN_OK;
}

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

static inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// grid of 256-thread blocks for a grid-stride loop over n elements, at most 16 blocks per SM
static inline int ew_grid(cgan_ctx* ctx, long long n) {
  long long b = (n + 255) / 256;
  long long cap = (long long)ctx->num_sms * 16;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

// round to the nearest TF32 value, ties away from zero
__device__ __forceinline__ float rna_tf32(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}

// the (leaky-)ReLU backward gate, TF's rule: with leak != 0 (leaky ReLU, tf.maximum(x, leak x), whose gradient goes to
// x on ties) v passes where x >= 0, -0 included; with leak 0 (ReLU, ReluGrad) where x > 0.  Elsewhere v is scaled by
// leak.  x: the activation's input or output (same sign).  Both rules are one comparison x > relu_gate_threshold(leak):
// x >= 0 is x > -2^-149, the negative float nearest to zero (the library is built without flush-to-zero).
__host__ __device__ __forceinline__ float relu_gate_threshold(float leak) { return leak != 0.f ? -0x1p-149f : 0.f; }
__device__ __forceinline__ float relu_gate(float x, float v, float leak) {
  return x > relu_gate_threshold(leak) ? v : leak * v;
}

// element i of the counter-based uniform [0, 1) stream (cgan_random_uniform): SplitMix64 of (seed, i + 1), 24 mantissa bits
__device__ __forceinline__ float splitmix_uniform(unsigned long long seed, unsigned long long i) {
  unsigned long long z = seed + 0x9E3779B97F4A7C15ull * (i + 1ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum; result valid in all threads. `sh` must hold 32 floats.
__device__ __forceinline__ float block_sum(float v, float* sh) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  int nw = (blockDim.x + 31) >> 5;
  float r = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.f;
  if (w == 0) {
    r = warp_sum(r);
    if (lane == 0) sh[0] = r;
  }
  __syncthreads();
  r = sh[0];
  return r;
}

// ---- tap lists of the tensor-core convolutions --------------------------------------------------------------------
// Tap (kh, kw) of a convolution d multiplies the HWIO weight slice kh * d->kw + kw.  Its signed offset per dimension is
// t = sign * (k - pad): sign +1 where the forward convolution reads its input relative to the output pixel, -1 for the
// adjoint (the input gradient reads dy relative to dx).  On a stride-2 grid t splits into t = 2 * half + parity:
//   TAP_DIRECT  offset t, view 0 (stride 1)
//   TAP_VIEW    offset half into view 2 * parity_h + parity_w: the operand is read through its four parity phases
//   TAP_PHASE   offset -half, view = output phase 2 * parity_h + parity_w: output pixel 2i + parity reads pixel i - half
constexpr int CGAN_TC_MAX_TAPS = 32;
enum TapRule { TAP_DIRECT, TAP_VIEW, TAP_PHASE };

struct ConvTaps {
  int ntaps;
  int off_h[CGAN_TC_MAX_TAPS], off_w[CGAN_TC_MAX_TAPS], wtap[CGAN_TC_MAX_TAPS], view[CGAN_TC_MAX_TAPS];
  int nphases;              // > 1: the list is grouped by output phase, phase ph owning taps [ph_tap0[ph], ph_tap0[ph + 1])
  int ph_tap0[5];
};

// false when the kernel has more taps than a list holds
static inline bool conv_taps(const cgan_conv_desc* d, int sign, TapRule rule, ConvTaps* t) {
  if (d->kh * d->kw > CGAN_TC_MAX_TAPS) return false;
  t->ntaps = 0;
  t->nphases = 1;
  for (int kh = 0; kh < d->kh; ++kh)
    for (int kw = 0; kw < d->kw; ++kw) {
      const int th = sign * (kh - d->pad_t), tw = sign * (kw - d->pad_l), a = th & 1, b = tw & 1;
      const int i = t->ntaps++;
      t->wtap[i] = kh * d->kw + kw;
      if (rule == TAP_DIRECT) {
        t->off_h[i] = th; t->off_w[i] = tw; t->view[i] = 0;
      } else {
        const int s = rule == TAP_VIEW ? 1 : -1;
        t->off_h[i] = s * (th - a) / 2; t->off_w[i] = s * (tw - b) / 2; t->view[i] = a * 2 + b;
      }
    }
  return true;
}

// TAP_PHASE taps grouped by output phase (in phase order, each phase in kernel order); false on an empty phase
static inline bool conv_taps_by_phase(const cgan_conv_desc* d, int sign, ConvTaps* t) {
  ConvTaps all;
  if (!conv_taps(d, sign, TAP_PHASE, &all)) return false;
  t->ntaps = 0;
  t->nphases = 4;
  for (int ph = 0; ph < 4; ++ph) {
    t->ph_tap0[ph] = t->ntaps;
    for (int i = 0; i < all.ntaps; ++i) {
      if (all.view[i] != ph) continue;
      const int j = t->ntaps++;
      t->off_h[j] = all.off_h[i]; t->off_w[j] = all.off_w[i]; t->wtap[j] = all.wtap[i]; t->view[j] = 0;
    }
    if (t->ntaps == t->ph_tap0[ph]) return false;
  }
  t->ph_tap0[4] = t->ntaps;
  return true;
}

// ---- activation operand of the wgmma kernels: `nviews` (1 or 4) NHWC views [n, h, w, ch] of `in` ---------------------
struct TcView {
  const float* in;
  int nviews;
  long long view_off[4];              // view v starts at in + view_off[v]
  long long sw, sh, sn;               // pixel strides (floats)
  int n, h, w, ch;
  int phase_h, phase_w;               // > 0: the four views are the parity phases of a phase_h x phase_w tensor
  int tf32;                           // the operand already holds TF32-representable values: no rounding in shared memory
};

// dense NHWC operand [n, h, w, c]
static inline void tc_in_dense(TcView* a, const float* x, int n, int h, int w, int ch) {
  a->in = x; a->nviews = 1; a->view_off[0] = 0;
  a->sw = ch; a->sh = (long long)w * ch; a->sn = (long long)h * w * ch;
  a->n = n; a->h = h; a->w = w; a->ch = ch;
}
// dense NHWC [n, H, W, c] read through its four parity phases: view 2a + b holds the pixels (2i + a, 2j + b)
static inline void tc_in_phases(TcView* a, const float* x, int n, int H, int W, int ch) {
  a->in = x; a->nviews = 4;
  for (int v = 0; v < 4; ++v) a->view_off[v] = ((long long)(v >> 1) * W + (v & 1)) * ch;
  a->sw = 2ll * ch; a->sh = 2ll * W * ch; a->sn = (long long)H * W * ch;
  a->n = n; a->h = (H + 1) / 2; a->w = (W + 1) / 2; a->ch = ch;
  a->phase_h = H; a->phase_w = W;
}

// ---- launch descriptor of the wgmma implicit-GEMM convolution (cgan_conv_tc, conv_tc.cu) ----------------------------
//   out[base + n*s_n + y*s_h + x*s_w + col] = epilogue(sum_{tap, k} a.view[tap][n, y + off_h, x + off_w, k] * W[wtap][col][k])
// for every output pixel (n, y, x), y < gh, x < gw.  Zero-initialise, then fill through the helpers below.
struct TcConv {
  TcView a;                           // activation operand, k = its channels
  int gh, gw;                         // output pixel grid
  // weights [taps_total][a.ch][ncols] (transpose_w = 1) or [taps_total][ncols][a.ch] (transpose_w = 0)
  const float* wsrc;
  int taps_total, transpose_w, ncols;
  int wimg_stride;                    // != 0: batched GEMM, image i multiplies weight slice wtap + i * wimg_stride
  ConvTaps taps;                      // views index the operand's views; with taps.nphases > 1 phase ph writes at ph_base[ph]
  // output
  float* out;
  long long s_n, s_h, s_w, base;
  long long ph_base[4];
  int ph_h[4], ph_w[4];               // > 0: phase ph stores only rows < ph_h[ph], columns < ph_w[ph] (0: the whole grid)
  // epilogue: + bias[col] + residual, then ReLU or the (leaky-)ReLU backward gate out = relu_gate(mask, v, mask_leak),
  // then TF32 rounding of the stored value
  const float* bias;
  const float* residual;
  const float* mask;
  float mask_leak;
  int relu, round_out;
};

// dense NHWC output over an h x w grid, rows of `ld` floats
static inline void tc_out_dense(TcConv* c, float* y, int h, int w, int ld) {
  c->out = y; c->gh = h; c->gw = w;
  c->s_w = ld; c->s_h = (long long)w * ld; c->s_n = (long long)h * w * ld; c->base = 0;
}
// dense NHWC [.., H, W, c] written through its parity phases: a ceil(H/2) x ceil(W/2) grid, phase 2a + b at pixel
// (2i + a, 2j + b).  Phase a holds the rows 2i + a < H, (H - a + 1) / 2 of them: for odd H the odd phases are one row
// short, and the epilogue stores nothing past a phase's own extent.
static inline void tc_out_phases(TcConv* c, float* y, int H, int W, int ch) {
  c->out = y; c->gh = (H + 1) / 2; c->gw = (W + 1) / 2;
  c->s_w = 2ll * ch; c->s_h = 2ll * W * ch; c->s_n = (long long)H * W * ch; c->base = 0;
  for (int v = 0; v < 4; ++v) {
    c->ph_base[v] = ((long long)(v >> 1) * W + (v & 1)) * ch;
    c->ph_h[v] = (H - (v >> 1) + 1) / 2; c->ph_w[v] = (W - (v & 1) + 1) / 2;
  }
}
// the whole epilogue of `ep` (null: none) and whether the activation operand is already TF32-rounded
static inline void tc_set_epilogue(TcConv* c, const cgan_conv_epilogue* ep, bool in_tf32) {
  c->a.tf32 = in_tf32 ? 1 : 0;
  if (!ep) return;
  c->bias = ep->bias; c->residual = ep->residual; c->mask = ep->mask; c->mask_leak = ep->mask_leak;
  c->relu = (ep->flags & CGAN_CONV_RELU) ? 1 : 0;
  c->round_out = (ep->flags & CGAN_CONV_ROUND_OUT) ? 1 : 0;
}

// Does `ep` still need a cgan_conv_post_epilogue pass after a kernel that applied only the bias (and the ReLU when
// relu_fused)?
static inline bool ep_needs_post(const cgan_conv_epilogue* ep, bool relu_fused) {
  return ep && (ep->residual || ep->mask || (ep->flags & CGAN_CONV_ROUND_OUT) || (!relu_fused && (ep->flags & CGAN_CONV_RELU)));
}

// ---- launch descriptor of the wgmma filter-gradient kernel (cgan_wgrad_tc, wgrad_tc.cu) -----------------------------
//   dw[wtap][ci][co] = sum_{n, y < dy.h, x < dy.w}  x.view[ax][n, y + off_h, x + off_w, ci] * dy.view[by][n, y, x, co]
// for every tap, with (ax, by) = (taps.view, 0), or (0, taps.view) when taps_view_dy: the pixel grid is that of dy's
// views.  Zero-initialise, then fill.
struct TcWgrad {
  TcView x;              // 1 view, or the four stride-2 parity phases (each of the grid's size)
  TcView dy;             // 1 view over the grid, or the four sub-pixel phases of the gradient of a zero-inserted input
  ConvTaps taps;
  int taps_view_dy;      // taps.view indexes dy's views (zero-inserted input) instead of x's (stride 2)
  int taps_total;        // dw holds taps_total slices [x.ch][dy.ch]
  float* dw;
  int per_image;         // per-image A^T B (one tap): dw slice i sums over image n = i only, stored with no reduce pass
};

int cgan_conv_tc(cgan_ctx* ctx, const TcConv& c);
// geometry the tensor-core convolution accepts for a stride-1 contraction
bool cgan_tc_shape_ok(int n, int h, int w, int kdim, int ncols);
int cgan_wgrad_tc(cgan_ctx* ctx, const TcWgrad& g);
// the filter-gradient kernel's own limits (box geometry, channel tiles, taps, alignment); routing policy is the caller's
bool cgan_wgrad_tc_fits(const TcWgrad& g);

// internal (C++ linkage) entry points shared between translation units
// gemm.cu
int cgan_conv2d_fwd_simt(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* w, const float* bias, float* y,
                         int relu, int ldy);
int cgan_conv2d_dgrad_simt(cgan_ctx*, const cgan_conv_desc*, const float* dy, const float* w, float* dx);
int cgan_conv2d_wgrad_simt(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, float* dw);
int cgan_gemm_batched_simt(cgan_ctx* ctx, int ta, int tb, int m, int n, int k, float alpha, const float* a, int lda,
                           int64_t sa, const float* b, int ldb, int64_t sb, float beta, float* c, int ldc, int64_t sc, int batch);
// out[i] = sum_{z < splits} part[z * n + i], summed in the order z = 0, 1, ... (deterministic split-K)
int cgan_splitk_reduce(cgan_ctx* ctx, float* out, const float* part, long long n, int splits);
// pointwise.cu
int cgan_conv_post_epilogue(cgan_ctx* ctx, float* y, int64_t rows, int c, int ld, const float* residual, const float* mask,
                            float mask_leak, int relu, int round_out);
int cgan_upsample1x1_bias_phases(cgan_ctx* ctx, float* out, const float* bias, int n, int oh, int ow, int c);
// thin.cu: exact-fp32 streaming kernels for image-side (<= 4 channel) convolutions
bool cgan_fwd_thin_ok(const cgan_conv_desc* d);
int cgan_fwd_thin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, float* y, int relu,
                  int ldy, int round_out);
bool cgan_fwd_thin3_ok(const cgan_conv_desc* d);
bool cgan_pw_thin_ok(const cgan_conv_desc* d);
int cgan_fwd_pw_thin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, float* y,
                     const float* residual, int relu, int ldy, int round_out);
bool cgan_wgrad_thin_ok(const cgan_conv_desc* d);
int cgan_wgrad_thin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, float* dw);
// thin_tc.cu: image-side convolutions through a 32-wide patch tensor on the tensor cores
bool cgan_thin_tc_cin_ok(cgan_ctx* ctx, const cgan_conv_desc* d);
bool cgan_thin_tc_wgrad_cin_ok(cgan_ctx* ctx, const cgan_conv_desc* d);
bool cgan_thin_tc_dgrad_cin_ok(cgan_ctx* ctx, const cgan_conv_desc* d);
bool cgan_thin_tc_cout_ok(cgan_ctx* ctx, const cgan_conv_desc* d);
bool cgan_thin_tc_wgrad_cout_ok(cgan_ctx* ctx, const cgan_conv_desc* d);
int cgan_thin_tc_fwd_cin(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* w, const cgan_conv_epilogue* ep, float* y);
int cgan_thin_tc_wgrad_cin(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* dy, int dy_tf32, float* dw);
int cgan_thin_tc_dgrad_cin(cgan_ctx*, const cgan_conv_desc*, const float* dy, const float* w, const cgan_conv_epilogue* ep, float* dx);
int cgan_thin_tc_fwd_cout(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* w, const cgan_conv_epilogue* ep, float* y);
int cgan_thin_tc_dgrad_cout(cgan_ctx*, const cgan_conv_desc*, const float* dy, const float* w, const cgan_conv_epilogue* ep, float* dx);
int cgan_thin_tc_wgrad_cout(cgan_ctx*, const cgan_conv_desc*, const float* x, const float* dy, int x_tf32, float* dw);
