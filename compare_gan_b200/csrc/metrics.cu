// FID statistics accumulator and the Inception pre-processing resize.
// Replaces: the covariance/mean part of tfgan.eval.frechet_classifier_distance_from_activations
// (metrics/fid_score.py:49-51) and tfgan.eval.preprocess_image (eval_utils.py:170-175).
#include "common.cuh"
#include "resize.cuh"

namespace {

// sumxxT[i,j] += sum_n act[n,i]*act[n,j] in float64.  One 16x16 output tile per block; the n loop is
// staged through shared memory so each activation row segment is read once per tile pair.
constexpr int CT = 16, CN = 32;
__global__ void cov_accumulate_kernel(const float* __restrict__ act, int n, int d, double* __restrict__ sum,
                                      double* __restrict__ sxx) {
  __shared__ float ai[CN][CT + 1], aj[CN][CT + 1];
  const int i0 = blockIdx.y * CT, j0 = blockIdx.x * CT;
  const int tx = threadIdx.x % CT, ty = threadIdx.x / CT;
  double acc = 0.0, accs = 0.0;
  for (int n0 = 0; n0 < n; n0 += CN) {
    for (int e = threadIdx.x; e < CN * CT; e += blockDim.x) {
      int r = e / CT, c = e % CT;
      ai[r][c] = (n0 + r < n && i0 + c < d) ? act[(long long)(n0 + r) * d + i0 + c] : 0.f;
      aj[r][c] = (n0 + r < n && j0 + c < d) ? act[(long long)(n0 + r) * d + j0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int r = 0; r < CN; ++r) {
      acc += (double)ai[r][ty] * (double)aj[r][tx];
      if (blockIdx.y == 0 && ty == 0) accs += (double)aj[r][tx];
    }
    __syncthreads();
  }
  if (i0 + ty < d && j0 + tx < d) sxx[(long long)(i0 + ty) * d + j0 + tx] += acc;
  if (blockIdx.y == 0 && ty == 0 && j0 + tx < d) sum[j0 + tx] += accs;
}

// tf.image.resize_bilinear, align_corners=False (legacy TF1 kernel: src = dst * scale, no half-pixel offset)
__global__ void resize_bilinear_kernel(float* __restrict__ y, const float* __restrict__ x, int n, int h, int w, int c,
                                       int oh, int ow, int incep) {
  long long tot = (long long)n * oh * ow * c;
  float sh = (float)h / (float)oh, sw = (float)w / (float)ow;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (long long)gridDim.x * blockDim.x) {
    int ch = (int)(i % c);
    long long t = i / c;
    int ox = (int)(t % ow); t /= ow;
    int oy = (int)(t % oh);
    long long b = t / oh;
    const TfBilinearTap ty = tf_bilinear_tap<false>(oy, sh, h), tx = tf_bilinear_tap<false>(ox, sw, w);
    const float* p = x + b * h * w * c + ch;
    float v = tf_bilinear<false>(p[((long long)ty.lo * w + tx.lo) * c], p[((long long)ty.lo * w + tx.hi) * c],
                                 p[((long long)ty.hi * w + tx.lo) * c], p[((long long)ty.hi * w + tx.hi) * c], tx.lerp, ty.lerp);
    if (incep) v = (v * 255.0f - 128.0f) / 128.0f;
    y[i] = v;
  }
}

}  // namespace

int cgan_cov_accumulate(cgan_ctx* ctx, const float* act, int n, int d, double* sum, double* sumxxT) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, act && sum && sumxxT && n > 0 && d > 0, "bad argument");
  dim3 grid(cdiv(d, CT), cdiv(d, CT));
  cov_accumulate_kernel<<<grid, CT * CT, 0, ctx->stream>>>(act, n, d, sum, sumxxT);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_resize_bilinear(cgan_ctx* ctx, float* y, const float* x, int n, int h, int w, int c, int oh, int ow, int incep) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, y && x && n > 0 && h > 0 && w > 0 && c > 0 && oh > 0 && ow > 0, "bad argument");
  long long tot = (long long)n * oh * ow * c;
  long long b = (tot + 255) / 256, cap = (long long)ctx->num_sms * 16;
  resize_bilinear_kernel<<<(int)(b > cap ? cap : b), 256, 0, ctx->stream>>>(y, x, n, h, w, c, oh, ow, incep);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}
