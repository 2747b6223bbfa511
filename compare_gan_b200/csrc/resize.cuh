// TF1's legacy bilinear resize (tf.image.resize_bilinear / tf.image.resize_images, align_corners = False), shared by the
// Inception pre-processing resize (metrics.cu) and the data set transforms (image_transform.cu): along each axis
// src = dst * (in / out) with no half-pixel offset, lo = floor(src), hi = min(lo + 1, in - 1), lerp = src - lo; then
// top = tl + (tr - tl) * lx, bot = bl + (br - bl) * lx, out = top + (bot - top) * ly in fp32.
// kExact = true keeps every operation a separately rounded fp32 operation, so the result equals a numpy float32
// restatement bit for bit; kExact = false leaves nvcc free to contract the multiply-adds (the Inception path's bits).
#pragma once

struct TfBilinearTap {
  int lo, hi;
  float lerp;
};

template <bool kExact>
__device__ __forceinline__ TfBilinearTap tf_bilinear_tap(int dst, float scale, int in) {
  TfBilinearTap t;
  const float src = kExact ? __fmul_rn((float)dst, scale) : dst * scale;
  t.lo = (int)floorf(src);
  t.hi = min(t.lo + 1, in - 1);
  t.lerp = kExact ? __fsub_rn(src, (float)t.lo) : src - t.lo;
  return t;
}

template <bool kExact>
__device__ __forceinline__ float tf_lerp(float a, float b, float l) {
  return kExact ? __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), l)) : a + (b - a) * l;
}

template <bool kExact>
__device__ __forceinline__ float tf_bilinear(float tl, float tr, float bl, float br, float lx, float ly) {
  const float top = tf_lerp<kExact>(tl, tr, lx), bot = tf_lerp<kExact>(bl, br, lx);
  return tf_lerp<kExact>(top, bot, ly);
}
