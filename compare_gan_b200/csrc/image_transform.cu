// Device half of the data set transforms (reference datasets.py:374-427, 440-532): a packed uint8 batch of crop windows
// (csrc/loader.cu, cgan_loader_create_transformed) -> float32 NHWC images in [0, 1] at the target resolution.  The host
// only picks the windows and copies their rows; the crop-or-pad canvas, the bilinear resize and the uint8 -> float
// conversion happen here, so the host->device copy carries uint8 windows instead of float images.
#include "common.cuh"
#include "resize.cuh"

namespace {

// One thread per output pixel, all c channels.  The kernel moves few bytes (a 128x128x3 output is 196 KB of float per
// image); the host->device copy of the windows dominates the transform's device time.
__global__ void crop_resize_u8_kernel(float* __restrict__ out, const uint8_t* __restrict__ packed,
                                      const cgan_crop_desc* __restrict__ desc, int n, int c, int r, int divide_after) {
  const long long tot = (long long)n * r * r;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % r);
    const long long t = i / r;
    const int oy = (int)(t % r), b = (int)(t / r);
    const cgan_crop_desc d = desc[b];
    const TfBilinearTap ty = tf_bilinear_tap<true>(oy, __fdiv_rn((float)d.canvas_h, (float)r), d.canvas_h);
    const TfBilinearTap tx = tf_bilinear_tap<true>(ox, __fdiv_rn((float)d.canvas_w, (float)r), d.canvas_w);
    // canvas rows / columns -> window rows / columns; -1 marks the zero padding of resize_image_with_crop_or_pad
    const int y0 = ty.lo - d.top, y1 = ty.hi - d.top, x0 = tx.lo - d.left, x1 = tx.hi - d.left;
    const bool iy0 = y0 >= 0 && y0 < d.h, iy1 = y1 >= 0 && y1 < d.h, ix0 = x0 >= 0 && x0 < d.w, ix1 = x1 >= 0 && x1 < d.w;
    const uint8_t* img = packed + d.offset;
    float* o = out + i * c;
    for (int ch = 0; ch < c; ++ch) {
      auto tap = [&](bool in, int y, int x) -> float {
        if (!in) return 0.f;
        const float v = (float)img[((long long)y * d.w + x) * c + ch];
        return divide_after ? v : __fdiv_rn(v, 255.0f);     // ImageNet: tf.cast(image, float32) / 255.0 before the resize
      };
      float v = tf_bilinear<true>(tap(iy0 && ix0, y0, x0), tap(iy0 && ix1, y0, x1), tap(iy1 && ix0, y1, x0),
                                  tap(iy1 && ix1, y1, x1), tx.lerp, ty.lerp);
      if (divide_after) v = __fdiv_rn(v, 255.0f);           // CelebA: resize the uint8 values, then / 255.0
      o[ch] = v;
    }
  }
}

}  // namespace

int cgan_crop_resize_u8(cgan_ctx* ctx, float* out, const uint8_t* packed, const cgan_crop_desc* desc, int n, int c, int r,
                        int divide_after) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, out && packed && desc && n > 0 && (c == 1 || c == 3) && r > 0 && (divide_after == 0 || divide_after == 1),
               "bad argument");
  const long long tot = (long long)n * r * r;
  const long long b = (tot + 255) / 256, cap = (long long)ctx->num_sms * 16;
  crop_resize_u8_kernel<<<(int)(b > cap ? cap : b), 256, 0, ctx->stream>>>(out, packed, desc, n, c, r, divide_after);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}
