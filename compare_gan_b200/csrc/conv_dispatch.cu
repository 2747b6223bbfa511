// Public conv entry points: choose between the exact-fp32 gather-GEMM (gemm.cu, math_mode 0) and the wgmma
// tensor-core implicit GEMM (conv_tc.cu, math_mode 1) according to the context's math mode and the shape.
#include "common.cuh"

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
  const bool ptr_ok = al16(x) && al16(y) && (!bias || al16(bias)) && (!ep || ((!ep->residual || al16(ep->residual)) &&
                                                                                  (!ep->mask || al16(ep->mask))));
  if (ctx->tc_thin && ptr_ok && ld_ok && al16(w) && !(d->kh == 1 && d->kw == 1)) {
    if (cgan_thin_tc_cin_ok(ctx, d)) {
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_fwd_cin(ctx, d, x, w, ep, y);
    }
    if (ldy == d->cout && cgan_thin_tc_cout_ok(ctx, d)) {
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_fwd_cout(ctx, d, x, w, ep, y);
    }
  }
  TcConv c = {};
  tc_in_dense(&c.a, x, d->n, d->h, d->w, d->cin);
  c.wsrc = w; c.taps_total = d->kh * d->kw; c.transpose_w = 1; c.ncols = d->cout;
  // a 1x1 kernel over a zero-inserted input (BigGAN's up-sampling shortcut): phase (0,0) is a plain 1x1 conv written to the
  // even pixels, the other three phases are bias only
  if (ctx->math_mode == 1 && d->stride == 1 && d->upsample && d->kh == 1 && d->kw == 1 && d->oh == 2 * d->h &&
      d->ow == 2 * d->w && d->pad_t == 0 && d->pad_l == 0 && d->cout % 4 == 0 &&
      cgan_tc_shape_ok(d->n, d->h, d->w, d->cin, d->cout) && ptr_ok) {
    c.taps.ntaps = 1;
    tc_out_phases(&c, y, d->oh, d->ow, d->cout);
    tc_set_epilogue(&c, nullptr, x_tf32);
    c.bias = bias;
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    int rc = cgan_conv_tc(ctx, c);
    if (rc) return rc;
    rc = cgan_upsample1x1_bias_phases(ctx, y, bias, d->n, d->oh, d->ow, d->cout);
    if (rc) return rc;
    if (ep_needs_post(ep, false))
      return cgan_conv_post_epilogue(ctx, y, (int64_t)d->n * d->oh * d->ow, d->cout, d->cout, ep->residual, ep->mask,
                                     ep->mask_leak, relu, (ep->flags & CGAN_CONV_ROUND_OUT) ? 1 : 0);
    return CGAN_OK;
  }
  tc_set_epilogue(&c, ep, x_tf32);
  if (ctx->math_mode == 1 && d->stride == 1 && d->kh * d->kw <= 32 && !(d->upsample && (d->kh < 2 || d->kw < 2)) &&
      (!d->upsample || (d->oh == 2 * d->h && d->ow == 2 * d->w)) && d->oh <= (d->upsample ? 2 * d->h : d->h) &&
      d->ow <= (d->upsample ? 2 * d->w : d->w) && cgan_tc_shape_ok(d->n, d->h, d->w, d->cin, d->cout) && ptr_ok &&
      !(d->upsample && d->cout % 4 != 0) && ld_ok) {
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    if (!d->upsample) {
      conv_taps(d, 1, TAP_DIRECT, &c.taps);
      tc_out_dense(&c, y, d->oh, d->ow, ldy);
      return cgan_conv_tc(ctx, c);
    }
    // conv over the zero-inserted 2x upsampled input (resnet_ops.py:35-56, 122-130) as four sub-pixel phases in one
    // launch (grid.z = phase): output pixel (2i+a, 2j+b) only sees the taps whose virtual input coordinate 2i+a+kh-pad is
    // even -> real pixel i+dh.
    if (!conv_taps_by_phase(d, -1, &c.taps))
      return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: empty sub-pixel phase%s", "cgan_conv2d_fwd");
    tc_out_phases(&c, y, d->oh, d->ow, d->cout);
    return cgan_conv_tc(ctx, c);
  }
  // stride 2 (SNDCGAN D, sndcgan.py:109-121): the input is read through its four (row, column) parity phases, each a
  // strided TMA view of the output's spatial size; tap (kh,kw) lands in phase ((kh-pad_t)&1, (kw-pad_l)&1).
  // Any size / SAME or VALID: phase a holds the rows 2r+a < H, i.e. (H-a+1)/2 of them (Inception's 35->17, 17->8).
  if (ctx->math_mode == 1 && d->stride == 2 && !d->upsample && d->kh * d->kw <= 32 && d->h >= 2 && d->w >= 2 &&
      (d->oh - 1) * 2 + d->kh - d->pad_t <= d->h + d->kh && cgan_tc_shape_ok(d->n, d->oh, d->ow, d->cin, d->cout) &&
      ptr_ok && ld_ok) {
    tc_in_phases(&c.a, x, d->n, d->h, d->w, d->cin);
    conv_taps(d, 1, TAP_VIEW, &c.taps);
    tc_out_dense(&c, y, d->oh, d->ow, ldy);
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    return cgan_conv_tc(ctx, c);
  }
  // exact-fp32 paths: residual / mask / rounding are applied by one extra pointwise pass
  bool post = ep_needs_post(ep, true);
  int rc;
  if (cgan_pw_thin_ok(d) && ptr_ok && al16(w) && ldy % 4 == 0 && !(ep && ep->mask)) {
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
  const bool ptr_ok = al16(dy) && al16(dx) && (!bias || al16(bias)) &&
                      (!ep || ((!ep->residual || al16(ep->residual)) && (!ep->mask || al16(ep->mask))));
  const bool geom = d->oh == (d->upsample ? 2 * d->h : d->h) && d->ow == (d->upsample ? 2 * d->w : d->w);
  // stride 2 (also tf.nn.conv2d_transpose of SNDCGAN's generator, arch_ops.py:588-589): input pixel 2i+a only receives
  // the taps with kh = a + pad_t (mod 2), from output row i + (a + pad_t - kh)/2 -> four input phases in one launch
  // (grid.z = phase), each writing a strided quarter of dx.  An odd H has ceil(H/2) output rows, and the odd phases of dx
  // are one row short of the even ones (tc_out_phases).
  const bool s2_phases = ctx->math_mode == 1 && d->stride == 2 && !d->upsample && d->kh * d->kw <= 16 && d->h >= 2 &&
                         d->w >= 2 && d->oh == (d->h + 1) / 2 && d->ow == (d->w + 1) / 2 && d->kh >= 2 && d->kw >= 2 &&
                         cgan_tc_shape_ok(d->n, d->oh, d->ow, d->cout, d->cin) && ptr_ok && d->cin % 4 == 0;
  if (ctx->tc_thin && ptr_ok && al16(w) && !(d->kh == 1 && d->kw == 1)) {
    if (cgan_thin_tc_cout_ok(ctx, d)) {          // dy has <= 4 channels (the generator's image conv)
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_dgrad_cout(ctx, d, dy, w, ep, dx);
    }
    // dx has <= 4 channels (gradient w.r.t. the discriminator's input image; the generator's stride-2 image layer).  A
    // stride-2 shape the phase kernel takes stays there.
    if (!s2_phases && cgan_thin_tc_dgrad_cin_ok(ctx, d)) {
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_thin_tc_dgrad_cin(ctx, d, dy, w, ep, dx);
    }
  }
  // dx[n,ih,iw,ci] = sum_{kh,kw,co} dy[n, oh, ow, co] * w[kh,kw,ci,co]: HWIO is already [tap][row=ci][k=co], i.e.
  // K-major for this contraction (no transpose).
  TcConv c = {};
  tc_in_dense(&c.a, dy, d->n, d->oh, d->ow, d->cout);
  c.wsrc = w; c.taps_total = d->kh * d->kw; c.transpose_w = 0; c.ncols = d->cin;
  tc_set_epilogue(&c, ep, dy_tf32);
  if (ctx->math_mode == 1 && d->stride == 1 && d->kh * d->kw <= 32 && geom &&
      cgan_tc_shape_ok(d->n, d->h, d->w, d->cout, d->cin) && ptr_ok) {
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    tc_out_dense(&c, dx, d->h, d->w, d->cin);
    if (!d->upsample) {
      conv_taps(d, -1, TAP_DIRECT, &c.taps);          // oh = ih + pad_t - kh
      return cgan_conv_tc(ctx, c);
    }
    // zero-inserted input: the real pixel ih sits at virtual row 2*ih; tap kh reaches output row oh = 2*ih + pad_t - kh,
    // i.e. sub-pixel phase a = (pad_t - kh) & 1 of dy at phase-row ih + (pad_t - kh - a)/2.  The four phases are four
    // strided TMA views of dy.
    tc_in_phases(&c.a, dy, d->n, d->oh, d->ow, d->cout);
    conv_taps(d, -1, TAP_VIEW, &c.taps);
    return cgan_conv_tc(ctx, c);
  }
  if (s2_phases) {
    ctx->last_path = CGAN_PATH_TCGEN05_TF32;
    if (!conv_taps_by_phase(d, 1, &c.taps))
      return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: empty phase%s", "cgan_conv2d_dgrad");
    tc_out_phases(&c, dx, d->h, d->w, d->cin);
    return cgan_conv_tc(ctx, c);
  }
  ctx->last_path = CGAN_PATH_SIMT_FP32;
  int rc = cgan_conv2d_dgrad_simt(ctx, d, dy, w, dx);
  if (rc) return rc;
  if (bias || ep_needs_post(ep, false)) {
    if (bias) {
      rc = cgan_bias_add(ctx, dx, dx, bias, (int64_t)d->n * d->h * d->w, d->cin);
      if (rc) return rc;
    }
    if (ep_needs_post(ep, false))
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
  if (ctx->tc_thin && d->n > 0 && d->kh * d->kw > 1 && al16(x) && al16(dy) && al16(dw)) {
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
  // The pixel loop runs over dy's grid: the input grid for stride 1 (also a zero-inserted input) and the output grid
  // for stride 2.  Stride 2: output (i, j) reads input row 2i + kh - pad_t = 2(i + dh) + a, i.e. parity phase view a
  // of X.  Zero-inserted input: output row 2i + a reads virtual row 2i + a + kh - pad_t, real only when even, from the
  // dY sub-pixel phase a = (pad_t - kh) & 1.
  if (ctx->math_mode == 1 && d->cin >= 64) {
    TcWgrad g = {};
    bool geom = false;
    if (d->stride == 2) {
      // an odd H gives ceil(H/2) output rows; the odd parity view of x is then one row short, and TMA zero-fills the
      // row past it exactly where SAME padding puts a zero (tc_in_phases)
      geom = !d->upsample && d->h >= 2 && d->w >= 2 && d->oh == (d->h + 1) / 2 && d->ow == (d->w + 1) / 2 &&
             conv_taps(d, 1, TAP_VIEW, &g.taps);
      tc_in_phases(&g.x, x, d->n, d->h, d->w, d->cin);
      tc_in_dense(&g.dy, dy, d->n, d->oh, d->ow, d->cout);
    } else if (d->stride == 1 && d->upsample) {
      geom = d->oh == 2 * d->h && d->ow == 2 * d->w && conv_taps(d, -1, TAP_PHASE, &g.taps);
      g.taps_view_dy = 1;
      tc_in_dense(&g.x, x, d->n, d->h, d->w, d->cin);
      tc_in_phases(&g.dy, dy, d->n, d->oh, d->ow, d->cout);
    } else if (d->stride == 1) {
      geom = d->oh == d->h && d->ow == d->w && conv_taps(d, 1, TAP_DIRECT, &g.taps);
      tc_in_dense(&g.x, x, d->n, d->h, d->w, d->cin);
      tc_in_dense(&g.dy, dy, d->n, d->oh, d->ow, d->cout);
    }
    g.x.tf32 = (flags & CGAN_CONV_IN_TF32) ? 1 : 0;
    g.dy.tf32 = (flags & CGAN_CONV_IN2_TF32) ? 1 : 0;
    g.taps_total = d->kh * d->kw;
    g.dw = dw;
    if (geom && cgan_wgrad_tc_fits(g)) {
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_wgrad_tc(ctx, g);
    }
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
      TcConv g = {};
      tc_in_dense(&g.a, a, batch, h, w, k);
      g.wsrc = b; g.taps_total = batch; g.transpose_w = nn ? 1 : 0; g.ncols = n; g.wimg_stride = 1;
      g.taps.ntaps = 1;                // one tap at offset 0: image i multiplies weight slice i
      tc_out_dense(&g, c, h, w, n);
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_conv_tc(ctx, g);
    }
  }
  if (ctx->math_mode == 1 && plain && ta && !tb && rows_as_grid(k, &h, &w) && lda == m && sa == (int64_t)k * m && ldb == n &&
      sb == (int64_t)k * n && ldc == n && sc == (int64_t)m * n && m >= 64 && n <= 256) {
    // C[i] = A[i]^T * B[i]: the reduction runs over the rows (pixels) -> the filter-gradient kernel, one image per CTA row
    TcWgrad g = {};
    tc_in_dense(&g.x, a, batch, h, w, m);
    tc_in_dense(&g.dy, b, batch, h, w, n);
    g.taps.ntaps = 1;                    // one tap at offset 0
    g.taps_total = 1;
    g.dw = c;
    g.per_image = 1;
    if (cgan_wgrad_tc_fits(g)) {
      ctx->last_path = CGAN_PATH_TCGEN05_TF32;
      return cgan_wgrad_tc(ctx, g);
    }
  }
  ctx->last_path = CGAN_PATH_SIMT_FP32;
  return cgan_gemm_batched_simt(ctx, ta, tb, m, n, k, alpha, a, lda, sa, b, ldb, sb, beta, c, ldc, sc, batch);
}

int cgan_gemm(cgan_ctx* ctx, int ta, int tb, int m, int n, int k, float alpha, const float* a, int lda, const float* b,
              int ldb, float beta, float* c, int ldc) {
  if (!ctx) return CGAN_ERR_ARG;
  ctx->last_path = CGAN_PATH_SIMT_FP32;
  return cgan_gemm_batched_simt(ctx, ta, tb, m, n, k, alpha, a, lda, 0, b, ldb, 0, beta, c, ldc, 0, 1);
}
