// Host-side input pipeline (SURVEY §8f row 4): the tf.data chain of ImageDatasetV2.train_input_fn
// (reference datasets.py:261-291) — repeat -> shuffle(buffer, seed) -> batch(drop_remainder) -> prefetch — as one
// producer thread that fills a ring of page-locked batch buffers while the GPU runs the previous cycle.  No device work
// happens here; the consumer (ModularGAN.set_inputs) issues the host->device copies and releases the slots afterwards.
//
// The transformed path (cgan_loader_create_transformed: ImageNet, CelebA and LSUN sources at their native sizes) picks each
// element's crop window on the host and packs only the window's rows, uint8, after a descriptor table; the device resizes
// them (csrc/image_transform.cu, cgan_crop_resize_u8).
#include <cuda_runtime.h>

#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/cgan_b200.h"

struct cgan_loader {
  const uint8_t* src_u8 = nullptr;
  const float* src_f32 = nullptr;
  const int32_t* src_labels = nullptr;
  int64_t n = 0;
  int64_t elems = 0;                 // h*w*c
  int batch = 0, ring = 0;
  std::vector<float*> images;        // ring slots
  std::vector<int32_t*> labels;
  bool pinned = false;
  float u8_to_unit[256];             // v / 255.0f, a true division as in TF (a multiply by 1/255 is 1 ulp off for some v)

  // transformed path: the element list (filtered source indices), the transform, and per slot one pinned area holding
  // [batch] descriptors followed by the packed window bytes
  bool transformed = false;
  cgan_image_source src{};
  cgan_image_transform tf{};
  std::vector<int32_t> list;
  uint64_t seed = 0;
  std::vector<uint8_t*> packed;
  std::vector<size_t> packed_cap;
  std::vector<int64_t> packed_used;

  // tf.data shuffle: a buffer of stream positions p of the infinite repeat() stream; position p is element p % n
  std::vector<int64_t> shuffle;
  int64_t next_source = 0;
  uint64_t rng_state = 0;

  // ring protocol: slots [tail, head) are filled or outstanding; produced counts fills, consumed counts next() calls,
  // released counts slots handed back.  produced - released <= ring.
  std::mutex mu;
  std::condition_variable cv_producer, cv_consumer;
  int64_t produced = 0, consumed = 0, released = 0;
  bool stop = false;
  bool failed = false;               // the producer could not fill a slot (err says why); next() fails from then on
  std::thread worker;
  char err[256] = {0};
};

namespace {

inline uint64_t splitmix64(uint64_t& s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// uniform integer in [0, bound) without modulo bias (rejection on the top of the range)
inline uint64_t uniform_below(uint64_t& s, uint64_t bound) {
  const uint64_t limit = UINT64_MAX - UINT64_MAX % bound;
  uint64_t r;
  do { r = splitmix64(s); } while (r >= limit);
  return r % bound;
}

int lfail(cgan_loader* L, int code, const char* msg) {
  if (L) snprintf(L->err, sizeof(L->err), "%s", msg);
  return code;
}

// the next stream position of the shuffled repeat() stream
inline int64_t next_position(cgan_loader* L) {
  if (L->shuffle.empty()) return L->next_source++;     // no shuffling: the plain repeat() stream
  const uint64_t slot = uniform_below(L->rng_state, L->shuffle.size());
  const int64_t p = L->shuffle[slot];
  L->shuffle[slot] = L->next_source++;   // replaced by the next input element
  return p;
}

void fill_slot(cgan_loader* L, int slot) {
  float* img = L->images[slot];
  int32_t* lab = L->labels[slot];
  for (int b = 0; b < L->batch; ++b) {
    const int64_t e = next_position(L) % L->n;
    float* dst = img + (int64_t)b * L->elems;
    if (L->src_u8) {
      const uint8_t* src = L->src_u8 + e * L->elems;
      for (int64_t i = 0; i < L->elems; ++i) dst[i] = L->u8_to_unit[src[i]];     // _parse_fn: tf.cast(image, float32) / 255.0
    } else {
      memcpy(dst, L->src_f32 + e * L->elems, (size_t)L->elems * sizeof(float));
    }
    lab[b] = L->src_labels ? L->src_labels[e] : 0;
  }
}

// ---- transformed path -------------------------------------------------------------------------------------------
// Every random draw of stream position p comes from its own SplitMix64 stream, keyed by (seed, p, stream id): the key
// is mix(mix(mix(seed) ^ p) ^ id), mix(x) being SplitMix64's output for state x.  Stream 0 draws the crop, stream 1 the
// random label.  TF's Philox streams are not restated: parity is of distribution, not of stream.
enum { kCropStream = 0, kLabelStream = 1 };

inline uint64_t mix(uint64_t x) { return splitmix64(x); }

inline uint64_t draw_key(uint64_t seed, int64_t p, uint64_t id) { return mix(mix(mix(seed) ^ (uint64_t)p) ^ id); }

// U[0, 1) with 24 random bits, as a float
inline float uniform01(uint64_t& s) { return (float)(splitmix64(s) >> 40) * (1.0f / 16777216.0f); }

// tf.image.sample_distorted_bounding_box of the whole image with aspect_ratio_range [1, 1], area_range [0.5, 1],
// max_attempts 100 (datasets.py:458-466), as TF 1.x's GenerateRandomCrop (core/kernels/sample_distorted_bounding_box_op.cc)
// reads; min_object_covered 0.1 always holds for a crop of at least half the image.  An attempt draws the side in the
// closed range [lrintf(sqrt(0.5 h w)), lrintf(sqrt(h w)) clamped to w and h], fixes the area up or down by one, is
// rejected when the square does not fit or its area leaves [0.5, 1] h w, and otherwise draws the offsets as
// Uniform(h - side), Uniform(w - side): in [0, h - side - 1], never the last position.  After 100 rejected attempts
// (images more elongated than 2:1) the crop is the whole image.  Returns the side (0 for the whole image).
int distorted_crop(int h, int w, uint64_t& s, int* y, int* x) {
  const float min_area = 0.5f * (float)w * (float)h, max_area = 1.0f * (float)w * (float)h;
  for (int attempt = 0; attempt < 100; ++attempt) {
    int side = (int)lrintf(std::sqrt(min_area));
    int max_side = (int)lrintf(std::sqrt(max_area));
    if (max_side > w) max_side = w;      // TF: the largest side whose rounded width fits, which for aspect 1 is w
    if (max_side > h) max_side = h;
    if (side >= max_side) side = max_side;
    if (side < max_side) side += (int)uniform_below(s, (uint64_t)(max_side - side + 1));
    int width = side;
    float area = (float)(width * side);
    if (area < min_area) { side += 1; width = side; area = (float)(width * side); }
    if (area > max_area) { side -= 1; width = side; area = (float)(width * side); }
    if (area < min_area || area > max_area || width > w || side > h || width <= 0 || side <= 0) continue;
    *y = side < h ? (int)uniform_below(s, (uint64_t)(h - side)) : 0;
    *x = width < w ? (int)uniform_below(s, (uint64_t)(w - width)) : 0;
    return side;
  }
  *y = *x = 0;
  return 0;
}

// the element's crop window (origin and extent in the source image) and its place on the canvas
void crop_window(const cgan_loader* L, int64_t p, int h, int w, cgan_crop_desc* d) {
  int cy = 0, cx = 0, wh = h, ww = w, ch = h, cw = w, top = 0, left = 0;
  uint64_t s = draw_key(L->seed, p, kCropStream);
  switch (L->tf.crop) {
    case CGAN_CROP_MIDDLE: {             // begin = int32(float32(h - side) / 2.0)
      const int side = std::min(h, w);
      cy = (int)((float)(h - side) / 2.0f);
      cx = (int)((float)(w - side) / 2.0f);
      wh = ww = ch = cw = side;
      break;
    }
    case CGAN_CROP_RANDOM: {             // begin = int32([h - side, w - side] * U[0,1)^2), truncated
      const int side = std::min(h, w);
      const float uy = uniform01(s), ux = uniform01(s);
      cy = (int)((float)(h - side) * uy);
      cx = (int)((float)(w - side) * ux);
      wh = ww = ch = cw = side;
      break;
    }
    case CGAN_CROP_DISTORTED: {
      const int side = distorted_crop(h, w, s, &cy, &cx);
      if (side > 0) wh = ww = ch = cw = side;
      break;
    }
    case CGAN_CROP_OR_PAD: {             // larger sides are centre-cropped at (size - target) // 2, smaller ones padded
      ch = L->tf.canvas_h;               // at (target - size) // 2
      cw = L->tf.canvas_w;
      if (h > ch) { cy = (h - ch) / 2; wh = ch; } else { top = (ch - h) / 2; }
      if (w > cw) { cx = (w - cw) / 2; ww = cw; } else { left = (cw - w) / 2; }
      break;
    }
    default: break;                      // CGAN_CROP_NONE: the whole image
  }
  d->h = wh; d->w = ww; d->canvas_h = ch; d->canvas_w = cw; d->top = top; d->left = left; d->crop_y = cy; d->crop_x = cx;
}

int64_t window_bound(const cgan_loader* L, int h, int w) {
  if (L->tf.crop == CGAN_CROP_OR_PAD) return (int64_t)std::min(h, L->tf.canvas_h) * std::min(w, L->tf.canvas_w) * L->src.c;
  return (int64_t)h * w * L->src.c;
}

bool grow_packed(cgan_loader* L, int slot, size_t bytes) {
  void* p = nullptr;
  if (L->pinned ? cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess : !(p = aligned_alloc(64, (bytes + 63) / 64 * 64)))
    return false;
  if (L->packed[slot]) { if (L->pinned) cudaFreeHost(L->packed[slot]); else free(L->packed[slot]); }
  L->packed[slot] = static_cast<uint8_t*>(p);
  L->packed_cap[slot] = bytes;
  return true;
}

bool fill_slot_transformed(cgan_loader* L, int slot) {
  const int c = L->src.c;
  std::vector<cgan_crop_desc> descs((size_t)L->batch);
  int32_t* lab = L->labels[slot];
  int64_t used = (int64_t)L->batch * sizeof(cgan_crop_desc);
  for (int b = 0; b < L->batch; ++b) {
    const int64_t p = next_position(L);
    const int32_t e = L->list[(size_t)(p % L->n)];
    const int64_t* row = L->src.index + 3 * (int64_t)e;
    cgan_crop_desc& d = descs[(size_t)b];
    memset(&d, 0, sizeof(d));
    d.position = p;
    d.element = e;
    crop_window(L, p, (int)row[1], (int)row[2], &d);
    d.offset = used;
    used += (int64_t)d.h * d.w * c;
    switch (L->tf.label) {
      case CGAN_LABEL_ZERO: lab[b] = 0; break;
      case CGAN_LABEL_RANDOM: {
        uint64_t s = draw_key(L->seed, p, kLabelStream);
        lab[b] = (int32_t)uniform_below(s, (uint64_t)L->tf.random_classes);
        break;
      }
      default: lab[b] = L->src.labels ? L->src.labels[e] : 0;
    }
  }
  // a batch that repeats large elements can need more than the slot was sized for: grow it (the slot is not outstanding)
  if ((size_t)used > L->packed_cap[slot] && !grow_packed(L, slot, (size_t)used + (size_t)used / 4)) {
    lfail(L, CGAN_ERR_WORKSPACE, "cgan_loader: could not grow a ring slot");
    return false;
  }
  uint8_t* base = L->packed[slot];
  memcpy(base, descs.data(), descs.size() * sizeof(cgan_crop_desc));
  for (const cgan_crop_desc& d : descs) {              // copy only the window's rows
    const int64_t* row = L->src.index + 3 * (int64_t)d.element;
    const int64_t w = row[2], rowbytes = (int64_t)d.w * c;
    const uint8_t* src = L->src.pixels + row[0] + ((int64_t)d.crop_y * w + d.crop_x) * c;
    uint8_t* dst = base + d.offset;
    for (int r = 0; r < d.h; ++r) memcpy(dst + r * rowbytes, src + r * w * c, (size_t)rowbytes);
  }
  L->packed_used[slot] = used;
  return true;
}

void producer(cgan_loader* L) {
  for (;;) {
    int slot;
    {
      std::unique_lock<std::mutex> lk(L->mu);
      L->cv_producer.wait(lk, [&] { return L->stop || L->produced - L->released < L->ring; });
      if (L->stop) return;
      slot = (int)(L->produced % L->ring);
    }
    // outside the lock: the slot is neither filled nor outstanding
    const bool ok = L->transformed ? fill_slot_transformed(L, slot) : (fill_slot(L, slot), true);
    {
      std::lock_guard<std::mutex> lk(L->mu);
      if (!ok) L->failed = true;
      else ++L->produced;
    }
    if (!ok) { L->cv_consumer.notify_all(); return; }
    L->cv_consumer.notify_one();
  }
}

// the shuffle buffer, the ring (float images or packed areas of `slot_bytes`, plus labels) and the producer thread
int start(cgan_loader* L, cgan_loader** out, int batch, int shuffle_buffer, uint64_t seed, int ring, size_t slot_bytes) {
  L->batch = batch;
  L->ring = ring;
  L->rng_state = seed;
  if (shuffle_buffer > 1) {              // tf.data fills the buffer with the first `buffer` elements of the stream
    L->shuffle.resize((size_t)shuffle_buffer);
    for (int i = 0; i < shuffle_buffer; ++i) L->shuffle[i] = L->next_source++;
  }
  int ndev = 0;
  L->pinned = cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0;
  if (!L->pinned) cudaGetLastError();    // clear the "no device" error: plain host memory is fine for a host pipeline
  const size_t lb = (size_t)batch * sizeof(int32_t);
  if (L->transformed) {
    L->packed.assign((size_t)ring, nullptr);
    L->packed_cap.assign((size_t)ring, 0);
    L->packed_used.assign((size_t)ring, 0);
  }
  for (int s = 0; s < ring; ++s) {
    void *pi = nullptr, *pl = nullptr;
    bool ok;
    if (L->transformed) {
      ok = grow_packed(L, s, slot_bytes);
    } else if (L->pinned) {
      ok = cudaHostAlloc(&pi, slot_bytes, cudaHostAllocPortable) == cudaSuccess;
    } else {
      ok = (pi = aligned_alloc(64, (slot_bytes + 63) / 64 * 64)) != nullptr;
    }
    if (ok) ok = L->pinned ? cudaHostAlloc(&pl, lb, cudaHostAllocPortable) == cudaSuccess : (pl = aligned_alloc(64, (lb + 63) / 64 * 64)) != nullptr;
    if (pi) L->images.push_back(static_cast<float*>(pi));
    if (pl) L->labels.push_back(static_cast<int32_t*>(pl));
    if (!ok) {
      const int code = L->pinned ? CGAN_ERR_CUDA : CGAN_ERR_WORKSPACE;
      cgan_loader_destroy(L);
      return code;
    }
  }
  L->worker = std::thread(producer, L);
  *out = L;
  return CGAN_OK;
}

// waits for the next filled slot; -1 (with err set) when the producer failed
int acquire_slot(cgan_loader* L) {
  std::unique_lock<std::mutex> lk(L->mu);
  if (L->consumed - L->released >= L->ring) {
    lfail(L, CGAN_ERR_ARG, "cgan_loader_next: every ring slot is outstanding; call cgan_loader_release first");
    return -1;
  }
  L->cv_consumer.wait(lk, [&] { return L->produced > L->consumed || L->failed; });
  if (L->produced <= L->consumed) return -1;
  const int slot = (int)(L->consumed % L->ring);
  ++L->consumed;
  return slot;
}

}  // namespace

extern "C" {

int cgan_loader_create(cgan_loader** out, const void* images, int src_dtype, const int32_t* labels, int64_t n, int h, int w,
                       int c, int batch, int shuffle_buffer, uint64_t seed, int ring) {
  if (!out || !images || n < 1 || h < 1 || w < 1 || c < 1 || batch < 1 || ring < 2 || (src_dtype != 0 && src_dtype != 1))
    return CGAN_ERR_ARG;
  cgan_loader* L = new cgan_loader();
  if (src_dtype == 0) L->src_u8 = static_cast<const uint8_t*>(images);
  else L->src_f32 = static_cast<const float*>(images);
  L->src_labels = labels;
  L->n = n;
  L->elems = (int64_t)h * w * c;
  for (int v = 0; v < 256; ++v) L->u8_to_unit[v] = (float)v / 255.0f;
  return start(L, out, batch, shuffle_buffer, seed, ring, (size_t)batch * L->elems * sizeof(float));
}

int cgan_loader_create_transformed(cgan_loader** out, const cgan_image_source* source, const cgan_image_transform* transform,
                                   int batch, int shuffle_buffer, uint64_t seed, int ring) {
  if (!out || !source || !transform || !source->pixels || !source->index || source->n < 1 || source->n > INT32_MAX ||
      (source->c != 1 && source->c != 3) || batch < 1 || ring < 2 || transform->crop < CGAN_CROP_NONE ||
      transform->crop > CGAN_CROP_OR_PAD || (transform->crop == CGAN_CROP_OR_PAD && (transform->canvas_h < 1 || transform->canvas_w < 1)) ||
      transform->label < CGAN_LABEL_SOURCE || transform->label > CGAN_LABEL_RANDOM ||
      (transform->label == CGAN_LABEL_RANDOM && transform->random_classes < 1))
    return CGAN_ERR_ARG;
  const cgan_image_source& S = *source;
  std::vector<int32_t> list;
  for (int64_t i = 0; i < S.n; ++i) {    // validate the table, then filter
    const int64_t off = S.index[3 * i], h = S.index[3 * i + 1], w = S.index[3 * i + 2];
    if (off < 0 || h < 1 || w < 1 || h > INT32_MAX || w > INT32_MAX || off > S.pixel_bytes ||
        h * w > (S.pixel_bytes - off) / S.c)
      return CGAN_ERR_ARG;
    if (transform->min_side > 0 && std::min(h, w) < transform->min_side) continue;
    if (transform->labeled_only && (!S.labels || S.labels[i] < 0)) continue;
    list.push_back((int32_t)i);
  }
  if (list.empty()) return CGAN_ERR_ARG;
  cgan_loader* L = new cgan_loader();
  L->transformed = true;
  L->src = S;
  L->tf = *transform;
  L->list.swap(list);
  L->n = (int64_t)L->list.size();
  L->seed = seed;
  // a slot holds the descriptors plus the largest window and `batch - 1` mean windows; a batch that needs more grows it
  int64_t largest = 0, total = 0;
  for (int32_t e : L->list) {
    const int64_t b = window_bound(L, (int)S.index[3 * (int64_t)e + 1], (int)S.index[3 * (int64_t)e + 2]);
    largest = std::max(largest, b);
    total += b;
  }
  const size_t bytes = (size_t)batch * sizeof(cgan_crop_desc) + (size_t)largest + (size_t)(batch - 1) * (size_t)(total / L->n);
  return start(L, out, batch, shuffle_buffer, seed, ring, bytes);
}

int cgan_loader_next(cgan_loader* L, const float** images, const int32_t** labels) {
  if (!L || !images || !labels) return CGAN_ERR_ARG;
  if (L->transformed) return lfail(L, CGAN_ERR_ARG, "cgan_loader_next: a transformed loader hands out packed batches (cgan_loader_next_packed)");
  const int slot = acquire_slot(L);
  if (slot < 0) return CGAN_ERR_ARG;
  *images = L->images[slot];
  *labels = L->labels[slot];
  return CGAN_OK;
}

int cgan_loader_next_packed(cgan_loader* L, const uint8_t** slot_data, int64_t* slot_bytes, const int32_t** labels) {
  if (!L || !slot_data || !slot_bytes || !labels) return CGAN_ERR_ARG;
  if (!L->transformed) return lfail(L, CGAN_ERR_ARG, "cgan_loader_next_packed: not a transformed loader");
  const int slot = acquire_slot(L);
  if (slot < 0) return L->failed ? CGAN_ERR_WORKSPACE : CGAN_ERR_ARG;
  *slot_data = L->packed[slot];
  *slot_bytes = L->packed_used[slot];
  *labels = L->labels[slot];
  return CGAN_OK;
}

int cgan_loader_release(cgan_loader* L, int count) {
  if (!L || count < 0) return CGAN_ERR_ARG;
  {
    std::lock_guard<std::mutex> lk(L->mu);
    if (L->released + count > L->consumed) return lfail(L, CGAN_ERR_ARG, "cgan_loader_release: more slots than outstanding");
    L->released += count;
  }
  L->cv_producer.notify_one();
  return CGAN_OK;
}

int cgan_loader_destroy(cgan_loader* L) {
  if (!L) return CGAN_ERR_ARG;
  {
    std::lock_guard<std::mutex> lk(L->mu);
    L->stop = true;
  }
  L->cv_producer.notify_all();
  if (L->worker.joinable()) L->worker.join();
  for (float* p : L->images) { if (L->pinned) cudaFreeHost(p); else free(p); }
  for (int32_t* p : L->labels) { if (L->pinned) cudaFreeHost(p); else free(p); }
  for (uint8_t* p : L->packed) { if (p) { if (L->pinned) cudaFreeHost(p); else free(p); } }
  delete L;
  return CGAN_OK;
}

const char* cgan_loader_last_error(cgan_loader* L) { return L ? L->err : "null loader"; }

}  // extern "C"
