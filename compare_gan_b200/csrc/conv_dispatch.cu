// Public conv entry points: choose between the exact-fp32 gather-GEMM (gemm.cu, math_mode 0) and the wgmma
// tensor-core implicit GEMM (conv_tc.cu, math_mode 1) according to the context's math mode and the shape.
#include "common.cuh"

bool cgan_tc_shape_ok(int n, int h, int w, int kdim, int ncols);
int cgan_conv_tc(cgan_ctx* ctx, const float* in, int nviews, const long long* view_off, long long in_sw, long long in_sh,
                 long long in_sn, int n, int h, int w, int gh, int gw, int kdim, const float* wsrc, int taps_total,
                 int transpose_w,
                 int ncols, int ntaps, const int* off_h, const int* off_w, const int* wtap, const int* amap,
                 const float* bias, float* out, long long s_n, long long s_h, long long s_w, long long base, int relu,
                 const int* view_phase_of = nullptr, int wimg_stride = 0, const TcExtra* ex = nullptr);
int cgan_tc_prep_weights(cgan_ctx* ctx, const float* wsrc, int taps_total, int transpose_w, int ncols, int kdim, float** out);
int cgan_conv_post_epilogue(cgan_ctx* ctx, float* y, int64_t rows, int c, int ld, const float* residual, const float* mask,
                            float mask_leak, int relu, int round_out);
bool cgan_fwd_thin_ok(const cgan_conv_desc* d);
int cgan_fwd_thin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, float* y, int relu,
                  int ldy, int round_out);
bool cgan_fwd_thin3_ok(const cgan_conv_desc* d);
bool cgan_pw_thin_ok(const cgan_conv_desc* d);
int cgan_fwd_pw_thin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, float* y,
                     const float* residual, int relu, int ldy, int round_out);
int cgan_wgrad_tc_batched(cgan_ctx* ctx, const float* a, const float* b, float* c, int batch, int h, int w, int k1, int k2);
bool cgan_wgrad_tc_ok(const cgan_conv_desc* d);
int cgan_wgrad_tc(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, float* dw, int x_tf32, int dy_tf32);
int cgan_conv2d_wgrad_simt(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, float* dw);
bool cgan_wgrad_thin_ok(const cgan_conv_desc* d);
int cgan_wgrad_thin(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, float* dw);

// image-side convolutions (<= 4 input or output channels) through a 32-wide patch tensor on the tensor cores (thin_tc.cu)
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

namespace {

inline TcExtra tc_extra(const cgan_conv_epilogue* ep, bool tf32_in) {
  TcExtra ex;
  memset(&ex, 0, sizeof(ex));
  ex.a_prerounded = tf32_in ? 1 : 0;
  if (ep) {
    ex.round_out = (ep->flags & CGAN_CONV_ROUND_OUT) ? 1 : 0;
    ex.residual = ep->residual; ex.mask = ep->mask; ex.mask_leak = ep->mask_leak;
  }
  return ex;
}
inline bool ep_has_post(const cgan_conv_epilogue* ep) {
  return ep && (ep->residual || ep->mask || (ep->flags & (CGAN_CONV_RELU | CGAN_CONV_ROUND_OUT)));
}
inline bool al16p(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

int cgan_conv2d_fwd(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, float* y) {
  return cgan_conv2d_fwd_act(ctx, d, x, w, bias, 0, y);
}

int cgan_conv2d_fwd_act(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, int act,
                        float* y) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, d, "null pointer");
  return cgan_conv2d_fwd_act_ld(ctx, d, x, w, bias, act, y, d->cout);
}

int cgan_conv2d_fwd_act_ld(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const float* bias, int act,
                           float* y, int ldy) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, act == 0 || act == CGAN_ACT_RELU, "act must be 0 or CGAN_ACT_RELU");
  cgan_conv_epilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.bias = bias;
  ep.flags = act == CGAN_ACT_RELU ? CGAN_CONV_RELU : 0;
  ep.ldy = ldy;
  return cgan_conv2d_fwd_ex(ctx, d, x, w, &ep, y);
}

int cgan_conv2d_fwd_ex(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* w, const cgan_conv_epilogue* ep,
                       float* y) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, d && x && w && y, "null pointer");
  const float* bias = ep ? ep->bias : nullptr;
  const int ldy = (ep && ep->ldy) ? ep->ldy : d->cout;
  const int relu = (ep && (ep->flags & CGAN_CONV_RELU)) ? 1 : 0;
  const bool x_tf32 = ep && (ep->flags & CGAN_CONV_IN_TF32);
  CGAN_REQUIRE(ctx, ldy >= d->cout, "ldy must be >= cout");
  CGAN_REQUIRE(ctx, ldy == d->cout || !d->upsample, "strided output is not available with upsample");
  const bool ld_ok = ldy == d->cout || ldy % 4 == 0;      // the tensor-core epilogue stores rows of float2 pairs (a multiple of 4 keeps them aligned)
  const bool ptr_ok = al16p(x) && al16p(y) && (!bias || al16p(bias)) && (!ep || ((!ep->residual || al16p(ep->residual)) &&
                                                                                  (!ep->mask || al16p(ep->mask))));
  TcExtra ex = tc_extra(ep, x_tf32);
  if (ctx->tc_thin && ptr_ok && ld_ok && al16p(w) && !(d->kh == 1 && d->kw == 1)) {
    if (cgan_thin_tc_cin_ok(ctx, d)) {
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_fwd_cin(ctx, d, x, w, ep, y);
    }
    if (ldy == d->cout && cgan_thin_tc_cout_ok(ctx, d)) {
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_fwd_cout(ctx, d, x, w, ep, y);
    }
  }
  // a 1x1 kernel over a zero-inserted input (BigGAN's up-sampling shortcut): phase (0,0) is a plain 1x1 conv written to the
  // even pixels, the other three phases are bias only
  if (ctx->math_mode == 1 && d->stride == 1 && d->upsample && d->kh == 1 && d->kw == 1 && d->oh == 2 * d->h &&
      d->ow == 2 * d->w && d->pad_t == 0 && d->pad_l == 0 && d->cout % 4 == 0 &&
      cgan_tc_shape_ok(d->n, d->h, d->w, d->cin, d->cout) && ptr_ok) {
    const long long zero = 0;
    const int o0 = 0, t0 = 0;
    TcExtra ex0;
    memset(&ex0, 0, sizeof(ex0));
    ex0.a_prerounded = ex.a_prerounded;
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    int rc = cgan_conv_tc(ctx, x, 1, &zero, d->cin, (long long)d->w * d->cin, (long long)d->h * d->w * d->cin, d->n, d->h,
                          d->w, d->h, d->w, d->cin, w, 1, 1, d->cout, 1, &o0, &o0, &t0, nullptr, bias, y,
                          (long long)d->oh * d->ow * d->cout, 2ll * d->ow * d->cout, 2ll * d->cout, 0, 0, nullptr, 0, &ex0);
    if (rc) return rc;
    rc = cgan_upsample1x1_bias_phases(ctx, y, bias, d->n, d->oh, d->ow, d->cout);
    if (rc) return rc;
    if (ep_has_post(ep))
      return cgan_conv_post_epilogue(ctx, y, (int64_t)d->n * d->oh * d->ow, d->cout, d->cout, ep->residual, ep->mask,
                                     ep->mask_leak, relu, ex.round_out);
    return CGAN_OK;
  }
  if (ctx->math_mode == 1 && d->stride == 1 && d->kh * d->kw <= 32 && !(d->upsample && (d->kh < 2 || d->kw < 2)) &&
      (!d->upsample || (d->oh == 2 * d->h && d->ow == 2 * d->w)) && d->oh <= (d->upsample ? 2 * d->h : d->h) &&
      d->ow <= (d->upsample ? 2 * d->w : d->w) && cgan_tc_shape_ok(d->n, d->h, d->w, d->cin, d->cout) && ptr_ok &&
      !(d->upsample && d->cout % 4 != 0) && ld_ok) {
    int oh[32], ow[32], wt[32];
    const long long zero = 0;
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    if (!d->upsample) {
      int nt = 0;
      for (int kh = 0; kh < d->kh; ++kh)
        for (int kw = 0; kw < d->kw; ++kw) {
          oh[nt] = kh - d->pad_t; ow[nt] = kw - d->pad_l; wt[nt] = kh * d->kw + kw; ++nt;
        }
      return cgan_conv_tc(ctx, x, 1, &zero, d->cin, (long long)d->w * d->cin, (long long)d->h * d->w * d->cin, d->n, d->h,
                          d->w, d->oh, d->ow, d->cin, w, d->kh * d->kw, 1, d->cout, nt, oh, ow, wt, nullptr, bias, y,
                          (long long)d->oh * d->ow * ldy, (long long)d->ow * ldy, ldy, 0, relu, nullptr, 0, &ex);
    }
    // conv over the zero-inserted 2x upsampled input (resnet_ops.py:35-56, 122-130) as four sub-pixel phases: output
    // pixel (2i+a, 2j+b) only sees the taps whose virtual input coordinate 2i+a+kh-pad is even -> real pixel i+dh.
    // The weights are prepared once for the four launches.
    // One launch (grid.z = phase), one weight preparation.
    int nt = 0;
    ex.nphases = 4;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        const int ph = a * 2 + b;
        ex.ph_tap0[ph] = nt;
        ex.ph_base[ph] = ((long long)a * d->ow + b) * d->cout;
        for (int kh = 0; kh < d->kh; ++kh) {
          int vh = a + kh - d->pad_t;
          if (vh & 1) continue;
          for (int kw = 0; kw < d->kw; ++kw) {
            int vw = b + kw - d->pad_l;
            if (vw & 1) continue;
            oh[nt] = vh / 2; ow[nt] = vw / 2;      // exact: vh, vw even (possibly negative)
            wt[nt] = kh * d->kw + kw; ++nt;
          }
        }
        if (nt == ex.ph_tap0[ph]) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: empty sub-pixel phase%s", "cgan_conv2d_fwd");
      }
    ex.ph_tap0[4] = nt;
    return cgan_conv_tc(ctx, x, 1, &zero, d->cin, (long long)d->w * d->cin, (long long)d->h * d->w * d->cin, d->n,
                        d->h, d->w, d->h, d->w, d->cin, w, d->kh * d->kw, 1, d->cout, nt, oh, ow, wt, nullptr, bias, y,
                        (long long)d->oh * d->ow * d->cout, 2ll * d->ow * d->cout, 2ll * d->cout, 0, relu, nullptr, 0, &ex);
  }
  // stride 2 (SNDCGAN D, sndcgan.py:109-121): the input is read through its four (row, column) parity phases, each a
  // strided TMA view of the output's spatial size; tap (kh,kw) lands in phase ((kh-pad_t)&1, (kw-pad_l)&1).
  // Any size / SAME or VALID: phase a holds the rows 2r+a < H, i.e. (H-a+1)/2 of them (Inception's 35->17, 17->8).
  if (ctx->math_mode == 1 && d->stride == 2 && !d->upsample && d->kh * d->kw <= 32 && d->h >= 2 && d->w >= 2 &&
      (d->oh - 1) * 2 + d->kh - d->pad_t <= d->h + d->kh && cgan_tc_shape_ok(d->n, d->oh, d->ow, d->cin, d->cout) &&
      ptr_ok && ld_ok) {
    int oh[32], ow[32], wt[32], am[32], nt = 0;
    const int hw[2] = {d->h, d->w};
    long long voff[4];
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) voff[a * 2 + b] = ((long long)a * d->w + b) * d->cin;
    for (int kh = 0; kh < d->kh; ++kh) {
      int th = kh - d->pad_t, a = th & 1;
      for (int kw = 0; kw < d->kw; ++kw) {
        int tw = kw - d->pad_l, b = tw & 1;
        oh[nt] = (th - a) / 2; ow[nt] = (tw - b) / 2; wt[nt] = kh * d->kw + kw; am[nt] = a * 2 + b; ++nt;
      }
    }
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    return cgan_conv_tc(ctx, x, 4, voff, 2ll * d->cin, 2ll * d->w * d->cin, (long long)d->h * d->w * d->cin, d->n,
                        (d->h + 1) / 2, (d->w + 1) / 2, d->oh, d->ow, d->cin, w, d->kh * d->kw, 1, d->cout, nt, oh, ow, wt, am,
                        bias, y, (long long)d->oh * d->ow * ldy, (long long)d->ow * ldy, ldy, 0, relu, hw, 0, &ex);
  }
  // exact-fp32 paths: residual / mask / rounding are applied by one extra pointwise pass
  bool post = ep && (ep->residual || ep->mask || (ep->flags & CGAN_CONV_ROUND_OUT));
  int rc;
  if (cgan_pw_thin_ok(d) && ptr_ok && al16p(w) && ldy % 4 == 0 && !(ep && ep->mask)) {
    // pointwise conv over <= 4 channels: one streaming kernel with residual add, ReLU and rounding fused
    ctx->last_path = CGAN_PATH_THIN_FP32;
    return cgan_fwd_pw_thin(ctx, d, x, w, bias, y, ep ? ep->residual : nullptr, relu, ldy,
                            (ep && (ep->flags & CGAN_CONV_ROUND_OUT)) ? 1 : 0);
  }
  if (cgan_fwd_thin_ok(d)) {
    ctx->last_path = CGAN_PATH_THIN_FP32;
    const bool fused = post && !ep->residual && !ep->mask && cgan_fwd_thin3_ok(d);   // ReLU + rounding in the 3x3 kernel itself
    if (fused) post = false;
    rc = cgan_fwd_thin(ctx, d, x, w, bias, y, post ? 0 : relu, ldy, fused ? 1 : 0);
  } else {
    ctx->last_path = CGAN_PATH_SIMT_FP32;
    rc = cgan_conv2d_fwd_simt(ctx, d, x, w, bias, y, post ? 0 : relu, ldy);
  }
  if (rc || !post) return rc;
  return cgan_conv_post_epilogue(ctx, y, (int64_t)d->n * d->oh * d->ow, d->cout, ldy, ep->residual, ep->mask, ep->mask_leak,
                                 relu, (ep->flags & CGAN_CONV_ROUND_OUT) ? 1 : 0);
}

int cgan_conv2d_dgrad(cgan_ctx* ctx, const cgan_conv_desc* d, const float* dy, const float* w, float* dx) {
  return cgan_conv2d_dgrad_ex(ctx, d, dy, w, nullptr, dx);
}

int cgan_conv2d_dgrad_ex(cgan_ctx* ctx, const cgan_conv_desc* d, const float* dy, const float* w, const cgan_conv_epilogue* ep,
                         float* dx) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, d && dy && w && dx, "null pointer");
  CGAN_REQUIRE(ctx, !ep || (!ep->ldy || ep->ldy == d->cin), "dgrad output is dense");
  const float* bias = ep ? ep->bias : nullptr;          // tf.nn.conv2d_transpose + bias (arch_ops.py:588-592)
  const int relu = (ep && (ep->flags & CGAN_CONV_RELU)) ? 1 : 0;
  const bool dy_tf32 = ep && (ep->flags & CGAN_CONV_IN_TF32);
  const bool ptr_ok = al16p(dy) && al16p(dx) && (!bias || al16p(bias)) &&
                      (!ep || ((!ep->residual || al16p(ep->residual)) && (!ep->mask || al16p(ep->mask))));
  TcExtra ex = tc_extra(ep, dy_tf32);
  const bool geom = d->oh == (d->upsample ? 2 * d->h : d->h) && d->ow == (d->upsample ? 2 * d->w : d->w);
  if (ctx->tc_thin && ptr_ok && al16p(w) && !(d->kh == 1 && d->kw == 1)) {
    if (cgan_thin_tc_cout_ok(ctx, d)) {          // dy has <= 4 channels (the generator's image conv)
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_dgrad_cout(ctx, d, dy, w, ep, dx);
    }
    if (cgan_thin_tc_dgrad_cin_ok(ctx, d)) {     // dx has <= 4 channels (gradient w.r.t. the discriminator's input image)
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_dgrad_cin(ctx, d, dy, w, ep, dx);
    }
  }
  if (ctx->math_mode == 1 && d->stride == 1 && d->kh * d->kw <= 32 && geom &&
      cgan_tc_shape_ok(d->n, d->h, d->w, d->cout, d->cin) && ptr_ok) {
    // dx[n,ih,iw,ci] = sum_{kh,kw,co} dy[n, oh, ow, co] * w[kh,kw,ci,co]: HWIO is already [tap][row=ci][k=co], i.e.
    // K-major for this contraction (no transpose).
    int oh[32], ow[32], wt[32], am[32], nt = 0;
    long long voff[4] = {0, 0, 0, 0};
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    if (!d->upsample) {
      // oh = ih + pad_t - kh
      for (int kh = 0; kh < d->kh; ++kh)
        for (int kw = 0; kw < d->kw; ++kw) {
          oh[nt] = d->pad_t - kh; ow[nt] = d->pad_l - kw; wt[nt] = kh * d->kw + kw; am[nt] = 0; ++nt;
        }
      return cgan_conv_tc(ctx, dy, 1, voff, d->cout, (long long)d->ow * d->cout, (long long)d->oh * d->ow * d->cout, d->n,
                          d->h, d->w, d->h, d->w, d->cout, w, d->kh * d->kw, 0, d->cin, nt, oh, ow, wt, am, bias, dx,
                          (long long)d->h * d->w * d->cin, (long long)d->w * d->cin, d->cin, 0, relu, nullptr, 0, &ex);
    }
    // zero-inserted input: the real pixel ih sits at virtual row 2*ih; tap kh reaches output row oh = 2*ih + pad_t - kh,
    // i.e. sub-pixel phase a = (pad_t - kh) & 1 of dy at phase-row ih + (pad_t - kh - a)/2.  The four phases are four
    // strided TMA views of dy.
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) voff[a * 2 + b] = ((long long)a * d->ow + b) * d->cout;
    for (int kh = 0; kh < d->kh; ++kh) {
      int th = d->pad_t - kh, a = th & 1;
      for (int kw = 0; kw < d->kw; ++kw) {
        int tw = d->pad_l - kw, b = tw & 1;
        oh[nt] = (th - a) / 2; ow[nt] = (tw - b) / 2; wt[nt] = kh * d->kw + kw; am[nt] = a * 2 + b; ++nt;
      }
    }
    return cgan_conv_tc(ctx, dy, 4, voff, 2ll * d->cout, 2ll * d->ow * d->cout, (long long)d->oh * d->ow * d->cout, d->n,
                        d->h, d->w, d->h, d->w, d->cout, w, d->kh * d->kw, 0, d->cin, nt, oh, ow, wt, am, bias, dx,
                        (long long)d->h * d->w * d->cin, (long long)d->w * d->cin, d->cin, 0, relu, nullptr, 0, &ex);
  }
  // stride 2 (also tf.nn.conv2d_transpose of SNDCGAN's generator, arch_ops.py:588-589): input pixel 2i+a only receives
  // the taps with kh = a + pad_t (mod 2), from output row i + (a + pad_t - kh)/2 -> four launches, one per input phase,
  // each writing a strided quarter of dx; the weights are prepared once.
  if (ctx->math_mode == 1 && d->stride == 2 && !d->upsample && d->kh * d->kw <= 16 && !(d->h & 1) && !(d->w & 1) &&
      d->oh == d->h / 2 && d->ow == d->w / 2 && d->kh >= 2 && d->kw >= 2 &&
      cgan_tc_shape_ok(d->n, d->oh, d->ow, d->cout, d->cin) && ptr_ok && d->cin % 4 == 0) {
    const long long zero = 0;
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    int oh[32], ow[32], wt[32], nt = 0;
    ex.nphases = 4;
    for (int a = 0; a < 2; ++a)
      for (int b = 0; b < 2; ++b) {
        const int ph = a * 2 + b;
        ex.ph_tap0[ph] = nt;
        ex.ph_base[ph] = ((long long)a * d->w + b) * d->cin;
        for (int kh = 0; kh < d->kh; ++kh) {
          int th = a + d->pad_t - kh;
          if (th & 1) continue;
          for (int kw = 0; kw < d->kw; ++kw) {
            int tw = b + d->pad_l - kw;
            if (tw & 1) continue;
            oh[nt] = th / 2; ow[nt] = tw / 2; wt[nt] = kh * d->kw + kw; ++nt;
          }
        }
        if (nt == ex.ph_tap0[ph]) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: empty phase%s", "cgan_conv2d_dgrad");
      }
    ex.ph_tap0[4] = nt;
    return cgan_conv_tc(ctx, dy, 1, &zero, d->cout, (long long)d->ow * d->cout, (long long)d->oh * d->ow * d->cout,
                        d->n, d->oh, d->ow, d->oh, d->ow, d->cout, w, d->kh * d->kw, 0, d->cin, nt, oh, ow, wt, nullptr,
                        bias, dx, (long long)d->h * d->w * d->cin, 2ll * d->w * d->cin, 2ll * d->cin, 0, relu, nullptr, 0, &ex);
  }
  ctx->last_path = CGAN_PATH_SIMT_FP32;
  int rc = cgan_conv2d_dgrad_simt(ctx, d, dy, w, dx);
  if (rc) return rc;
  if (bias || ep_has_post(ep)) {
    if (bias) {
      rc = cgan_bias_add(ctx, dx, dx, bias, (int64_t)d->n * d->h * d->w, d->cin);
      if (rc) return rc;
    }
    if (ep_has_post(ep))
      return cgan_conv_post_epilogue(ctx, dx, (int64_t)d->n * d->h * d->w, d->cin, d->cin, ep->residual, ep->mask,
                                     ep->mask_leak, relu, (ep->flags & CGAN_CONV_ROUND_OUT) ? 1 : 0);
  }
  return CGAN_OK;
}

int cgan_conv2d_wgrad(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, float* dw) {
  return cgan_conv2d_wgrad_ex(ctx, d, x, dy, 0, dw);
}

int cgan_conv2d_wgrad_ex(cgan_ctx* ctx, const cgan_conv_desc* d, const float* x, const float* dy, int flags, float* dw) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, d && x && dy && dw, "null pointer");
  if (ctx->tc_thin && d->n > 0 && d->kh * d->kw > 1 && al16p(x) && al16p(dy) && al16p(dw)) {
    if (cgan_thin_tc_wgrad_cin_ok(ctx, d)) {
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_wgrad_cin(ctx, d, x, dy, (flags & CGAN_CONV_IN2_TF32) ? 1 : 0, dw);
    }
    if (cgan_thin_tc_wgrad_cout_ok(ctx, d)) {
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_wgrad_cout(ctx, d, x, dy, (flags & CGAN_CONV_IN_TF32) ? 1 : 0, dw);
    }
  }
  if (d->n > 0 && d->cin > 0 && d->cout > 0 && d->kh > 0 && d->kw > 0 && d->stride > 0 && cgan_wgrad_thin_ok(d)) {
    ctx->last_path = CGAN_PATH_THIN_FP32;
    return cgan_wgrad_thin(ctx, d, x, dy, dw);      // exact fp32 streaming kernels for 3-channel image-side layers
  }
  if (ctx->math_mode == 1 && cgan_wgrad_tc_ok(d) && al16p(x) && al16p(dy) && al16p(dw)) {
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    return cgan_wgrad_tc(ctx, d, x, dy, dw, (flags & CGAN_CONV_IN_TF32) ? 1 : 0, (flags & CGAN_CONV_IN2_TF32) ? 1 : 0);
  }
  ctx->last_path = CGAN_PATH_SIMT_FP32;
  return cgan_conv2d_wgrad_simt(ctx, d, x, dy, dw);
}


// ---- batched GEMM on tensor cores (attention, arch_ops.py:744, 753 and their gradients) ------------------------------
// rows of each matrix are laid out as an h x w pixel grid so the conv tiling applies; m = h*w must be >= 128.
static bool rows_as_grid(int m, int* h, int* w) {
  if (m < 128) return false;
  for (int ww = 128; ww >= 8; ww >>= 1)
    if (m % ww == 0) { *w = ww; *h = m / ww; return true; }
  return false;
}

int cgan_gemm_batched(cgan_ctx* ctx, int ta, int tb, int m, int n, int k, float alpha, const float* a, int lda, int64_t sa,
                      const float* b, int ldb, int64_t sb, float beta, float* c, int ldc, int64_t sc, int batch) {
  if (!ctx) return CGAN_ERR_ARG;
  const bool plain = alpha == 1.0f && beta == 0.0f && batch > 1 && a && b && c &&
                     ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c)) & 15) == 0;
  int h, w;
  if (ctx->math_mode == 1 && plain && !ta && rows_as_grid(m, &h, &w) && lda == k && sa == (int64_t)m * k && ldc == n &&
      sc == (int64_t)m * n && k % 4 == 0 && k >= 8 && n % 4 == 0 && cgan_tc_shape_ok(batch, h, w, k, n)) {
    // C[i] = A[i] * op(B[i]):  A[i] rows = pixels, k = channels; B[i] is the per-image "weight" slice
    const bool nt = tb && ldb == k && sb == (int64_t)n * k;        // B[i] stored [n, k]  (K-major already)
    const bool nn = !tb && ldb == n && sb == (int64_t)k * n;       // B[i] stored [k, n]  (transposed by the prep kernel)
    if (nt || nn) {
      const long long zero = 0;
      const int o0 = 0;
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_conv_tc(ctx, a, 1, &zero, k, (long long)w * k, (long long)m * k, batch, h, w, h, w, k, b, batch, nn ? 1 : 0, n,
                          1, &o0, &o0, &o0, nullptr, nullptr, c, (long long)m * n, (long long)w * n, n, 0, 0, nullptr, 1);
    }
  }
  if (ctx->math_mode == 1 && plain && ta && !tb && rows_as_grid(k, &h, &w) && lda == m && sa == (int64_t)k * m && ldb == n &&
      sb == (int64_t)k * n && ldc == n && sc == (int64_t)m * n && m % 32 == 0 && m >= 64 && n % 4 == 0 && n <= 256 && k % 32 == 0) {
    // C[i] = A[i]^T * B[i]: the reduction runs over the rows (pixels) -> the filter-gradient kernel, one image per CTA row
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    return cgan_wgrad_tc_batched(ctx, a, b, c, batch, h, w, m, n);
  }
  ctx->last_path = CGAN_PATH_SIMT_FP32;
  return cgan_gemm_batched_simt(ctx, ta, tb, m, n, k, alpha, a, lda, sa, b, ldb, sb, beta, c, ldc, sc, batch);
}

int cgan_gemm(cgan_ctx* ctx, int ta, int tb, int m, int n, int k, float alpha, const float* a, int lda, const float* b,
              int ldb, float beta, float* c, int ldc) {
  return cgan_gemm_batched_simt(ctx, ta, tb, m, n, k, alpha, a, lda, 0, b, ldb, 0, beta, c, ldc, 0, 1);
}
