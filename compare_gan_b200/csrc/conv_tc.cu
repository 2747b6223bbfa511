// Warpgroup-MMA (wgmma, sm_90a) implicit-GEMM convolution — math_mode 1.
//
//   out[pixel, co] = sum_{tap, ci} in[pixel + off(tap), ci] * wt[tap][co][ci]        (+ bias[co])
//
// * A operand (activations, NHWC fp32): one TMA 4-D tiled load per (tap, 32-channel chunk) brings a
//   [images x rows x cols x 32ch] box = 128 pixels x 128 B straight into the 128B-swizzled K-major layout
//   the wgmma descriptor expects; TF SAME padding is the TMA out-of-bounds zero fill (negative coordinates),
//   so no im2col buffer and no padding pass exist.
// * B operand (weights): pre-rounded (round-to-nearest TF32) and laid out [tap][row][k] K-major by a small
//   prep kernel; TMA 3-D loads.
// * The fp32 activations are rounded to nearest TF32 IN SHARED MEMORY by the consumer warpgroups before their
//   MMAs read them — the tensor core would otherwise truncate the low 13 bits, a systematic -2^-11 relative bias per
//   product that accumulates through a 13-layer discriminator.
// * Warp roles: warps 0..7 = two consumer warpgroups, warpgroup g owning rows 64g..64g+63 of every 128-pixel tile:
//   (operand rounding,) wgmma m64nBNk8 (K = 8 per instruction, fp32 accumulators in registers), epilogue from the
//   accumulator fragments (+bias, residual, ReLU / mask, TF32 rounding); warp 8 = TMA producer.
//   Stages are released one k-block late (wgmma.wait_group 1), so the rounding of the next stage overlaps the MMAs.
// * The epilogue of a float2 launch goes through the stage ring (tile_epilogue_smem): after its last k-block the
//   producer goes on around the ring, one 32-column chunk of the CTA's tile per slot, TMA-loading the chunk of a residual
//   or ReLU mask (tensors of the output's geometry, far larger than L2 in a training step) where the launch has one.
//   The consumers write the finished chunk into the slot, and one thread TMA-stores it to the output.
//
// The same kernel serves forward and input-gradient convolutions (and the four sub-pixel phases of a
// conv over a zero-inserted 2x upsampled input): the host supplies, per tap, the input offset and the weight
// slice, and the output pixel strides.
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int TC_BM = 128;          // output pixels per CTA tile (two warpgroups x wgmma M = 64)
constexpr int TC_BK = 32;           // fp32 channels per k-block: 128 B = one swizzle row
constexpr int TC_MAX_STAGES = 4;
constexpr int TC_MAX_TAPS = 32;
constexpr int TC_CWARPS = 8;        // consumer warps (two warpgroups)
constexpr int TC_THREADS = 32 * TC_CWARPS + 32;     // + the TMA producer warp
constexpr int TC_A_BYTES = TC_BM * TC_BK * 4;     // 16 KB
constexpr int TC_WG_A_BYTES = TC_A_BYTES / 2;      // one warpgroup's 64 rows
constexpr int TC_ACC_COLS = 256;    // mt x bn accumulator columns per CTA: mt*bn/2 registers per consumer thread

struct TcParams {
  int ntaps, kchunks;               // k-blocks = ntaps * kchunks
  int off_h[TC_MAX_TAPS], off_w[TC_MAX_TAPS], wtap[TC_MAX_TAPS], amap[TC_MAX_TAPS];   // amap: which input view
  int bw, bh, bni;                  // tile box: bw*bh*bni == 128
  int tiles_w, tiles_h;             // tiles per image row / column
  int rows_used;                    // bw*bh*bni <= 128 pixel rows actually filled by the TMA box
  int img_n;                        // images of the pixel grid (tiles at the border hang over; those rows are not stored)
  int relu;                         // fused ReLU in the epilogue
  int vec2;                         // 1: every output row starts at an even element offset and cout is even (float2 stores)
  int round_a;                      // 1: round the activation tiles to nearest TF32 in shared memory (operand not pre-rounded)
  int round_out;                    // 1: store TF32-rounded outputs (the consumer is another tensor-core contraction)
  float mask_leak;                  // with `mask`: out = ref > mask_thr ? v : mask_leak * v  ((leaky-)ReLU backward fused into a dgrad)
  float mask_thr;                   // relu_gate_threshold(mask_leak): relu_gate with the threshold chosen once on the host
  const float* residual;            // optional tensor of the output's geometry added before the activation (residual blocks)
  const float* mask;                // optional tensor of the output's geometry: the (leaky-)ReLU input/output whose sign gates v
  int wimg_stride;                  // batched GEMM: weight slice = wtap + image * wimg_stride (tiles never span images)
  int bn;                           // wgmma N (multiple of 32, <= 256)
  int stages;                       // smem pipeline depth (2..4)
  int mt;                           // pixel tiles per CTA sharing one weight tile (mt x bn accumulator columns)
  int tiles_total;                  // tiles_w * tiles_h * tiles_n
  int cout;                         // valid output channels (row length of `out` pixels)
  long long s_n, s_h, s_w, base;    // output element strides / offset (floats)
  float* out;
  const float* bias;
  // sub-pixel phases merged into one launch (blockIdx.z): phase ph owns the taps [ph_tap0[ph], ph_tap0[ph+1]) and writes
  // at element offset ph_base[ph] (a convolution over a zero-inserted input, a stride-2 input gradient)
  int nphases;
  int ph_tap0[5];
  long long ph_base[4];
  int ph_h[4], ph_w[4];             // pixels phase ph stores: rows < ph_h[ph], columns < ph_w[ph] (odd stride-2 dx: unequal)
  // halo mode (conv_tc_halo_kernel): the taps come in `hg` groups of `hnv` vertically consecutive taps that share their
  // horizontal offset; one TMA box of bh + hnv - 1 rows serves all taps of a group (the vertical shift is a descriptor
  // offset of bw rows), so the activation operand crosses L2 -> smem `hg` times per channel chunk instead of hg * hnv
  int hg, hnv;
  int h_off_w[4], h_off_h0[4], h_wtap[4][4];
  int a_halo_bytes;                 // smem footprint of one tile's halo box (1024-aligned)
  int a_box_bytes;                  // bytes TMA writes per halo box
  int sa_stages, sb_stages;
  int ep_tma;                       // 1: the tile is staged in the stage ring and TMA-stored (tile_epilogue_smem)
  int ep_smem;                      // 1: with ep_tma, the residual or mask is prefetched into the ring as well
};

// up to four views of the input tensor (the sub-pixel phases of a 2x-upsampled gradient); plain convs use view 0.  The
// same holds views of the residual / mask and of the output, one per output phase.
struct AMaps { CUtensorMap m[4]; };


__device__ __forceinline__ void tc_tile_origin(const TcParams& p, int t, int& ow0, int& oh0, int& n0) {
  const int tw = t % p.tiles_w; t /= p.tiles_w;
  const int th = t % p.tiles_h;
  const int tn = t / p.tiles_h;
  ow0 = tw * p.bw; oh0 = th * p.bh; n0 = tn * p.bni;
}

__device__ __forceinline__ float epilogue_one(const TcParams& p, float v, int col, long long off) {
  if (p.bias) v += p.bias[col];
  if (p.residual) v += p.residual[off];
  if (p.relu) v = fmaxf(v, 0.f);
  if (p.mask) v = p.mask[off] > p.mask_thr ? v : p.mask_leak * v;
  if (p.round_out) v = rna_tf32(v);
  return v;
}

// Epilogue of one pixel tile from the accumulator fragment of this thread: rows m and m + 8 of the tile, columns
// 8j + 2 (lane % 4) + {0, 1}.  A quad of lanes writes 32 contiguous bytes of one output row.  Rows beyond the box (stale
// smem) and pixels outside the grid are computed but never stored.
template <int BN>
__device__ __forceinline__ void tile_epilogue(const TcParams& p, const float* acc, int tile, int nb0, int wg, int warp, int lane,
                                            long long out_base) {
  int ow0, oh0, n0;
  tc_tile_origin(p, tile, ow0, oh0, n0);
  const int c2 = (lane & 3) * 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = wg * 64 + (warp & 3) * 16 + (lane >> 2) + h * 8;
    const int wi = m % p.bw;
    const int hi = (m / p.bw) % p.bh;
    const int ni = m / (p.bw * p.bh);
    if (!(m < p.rows_used && n0 + ni < p.img_n && oh0 + hi < p.ph_h[blockIdx.z] && ow0 + wi < p.ph_w[blockIdx.z])) continue;
    const long long roff = out_base + (long long)(n0 + ni) * p.s_n + (long long)(oh0 + hi) * p.s_h +
                           (long long)(ow0 + wi) * p.s_w + nb0;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = j * 8 + c2;
      if (nb0 + c >= p.cout) continue;
      float2 v = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      const long long off = roff + c;
      if (p.vec2) {
        if (p.bias) { const float2 b = *reinterpret_cast<const float2*>(p.bias + nb0 + c); v.x += b.x; v.y += b.y; }
        if (p.residual) { const float2 r = *reinterpret_cast<const float2*>(p.residual + off); v.x += r.x; v.y += r.y; }
        if (p.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
        if (p.mask) {
          const float2 mv = *reinterpret_cast<const float2*>(p.mask + off);
          v.x = mv.x > p.mask_thr ? v.x : p.mask_leak * v.x; v.y = mv.y > p.mask_thr ? v.y : p.mask_leak * v.y;
        }
        if (p.round_out) { v.x = rna_tf32(v.x); v.y = rna_tf32(v.y); }
        *reinterpret_cast<float2*>(p.out + off) = v;
      } else {        // odd column count or odd row offsets (e.g. the 256->3 image conv): element by element
        p.out[off] = epilogue_one(p, v.x, nb0 + c, off);
        if (nb0 + c + 1 < p.cout) p.out[off + 1] = epilogue_one(p, v.y, nb0 + c + 1, off + 1);
      }
    }
  }
}

// The same epilogue for a float2 launch with at most one of residual / mask, staged through the stage ring: chunk cc
// (32 columns) of the tile is a [rows_used][32] box in the next slot, 128B-swizzled, rows in the tile's pixel order.
// The producer fills the slot with the chunk of the residual or mask, or just hands it over when there is none.  Each
// thread finishes its elements at their swizzled addresses (bias from shared memory; the arithmetic and its order are
// tile_epilogue's), and thread 0 stores the box with one TMA store through the output map of the CTA's phase.  The map
// clips the rows past the grid or the phase's extent and the columns past cout, so no element needs a predicate or a
// global address.  Thread 0 hands a slot back to the producer once the store that reads it has read it and a later
// chunk of this CTA needs it: after issuing the store of chunk k it waits for the store of chunk k - 1 (issued one
// chunk earlier, normally done reading by then) and releases that slot, so the producer can load chunk k - 1 + stages
// while chunk k + 1 is being finished.
template <int BN>
__device__ __forceinline__ void tile_epilogue_smem(const TcParams& p, const CUtensorMap* om, const float* acc, int tile,
                                                 int nb0, int wg, int warp, int lane, const uint8_t* smem, int stage_bytes,
                                                 uint64_t* full_bar, uint64_t* empty_bar, int& stage, uint32_t& phase,
                                                 int& chunk, int chunks, uint32_t bias_addr) {
  int ow0, oh0, n0;
  tc_tile_origin(p, tile, ow0, oh0, n0);
  const int c2 = (lane & 3) * 2;
  const int m0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const bool operand = p.residual || p.mask;
#pragma unroll
  for (int cc = 0; cc < BN / 32; ++cc) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t e_addr = smem_u32(smem + stage * stage_bytes);
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = cc * 4 + jj, c = j * 8 + c2;
      const float2 b = p.bias ? lds64(bias_addr + c * 4) : make_float2(0.f, 0.f);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t a = e_addr + sw128_offset(m0 + h * 8, jj * 8 + c2);
        float2 v = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        const float2 e = operand ? lds64(a) : make_float2(0.f, 0.f);
        if (p.bias) { v.x += b.x; v.y += b.y; }
        if (p.residual) { v.x += e.x; v.y += e.y; }
        if (p.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); }
        if (p.mask) { v.x = e.x > p.mask_thr ? v.x : p.mask_leak * v.x; v.y = e.y > p.mask_thr ? v.y : p.mask_leak * v.y; }
        if (p.round_out) { v.x = rna_tf32(v.x); v.y = rna_tf32(v.y); }
        sts64(a, v);
      }
    }
    fence_proxy_async();                       // the chunk's writes become visible to the TMA store
    named_bar(3, 32 * TC_CWARPS);
    if (threadIdx.x == 0) {
      tma_store_4d(om, e_addr, nb0 + cc * 32, ow0, oh0, n0);
      bulk_commit();
      bulk_wait_read<1>();                     // the store of chunk - 1 has read its slot
      if (chunk >= 1 && chunk - 1 + p.stages < chunks) mbar_arrive(&empty_bar[stage == 0 ? p.stages - 1 : stage - 1], 2);
    }
    ++chunk;
    if (++stage == p.stages) { stage = 0; phase ^= 1; }
  }
}

// CTAs per SM the register allocation has to allow.  The register file is split among the SM's four schedulers: two
// CTAs of nine warps put five warps on one of them, so each thread may hold at most 16384 / (5 x 32) -> 96 registers.
// At 100 registers the 128-column tile ran one CTA per SM although its shared memory fits two.
constexpr int tc_min_ctas(int bn, int mt) { return bn * mt <= 128 ? 2 : 1; }

// round this warpgroup's `bytes` of a tile (float4 per thread and sweep) to nearest TF32 in place
__device__ __forceinline__ void tc_round_smem(uint32_t base, int bytes, int q, int nthreads) {
#pragma unroll 4
  for (int i = q * 16; i < bytes; i += nthreads * 16) {
    float4 v = lds128(base + i);
    v.x = rna_tf32(v.x); v.y = rna_tf32(v.y); v.z = rna_tf32(v.z); v.w = rna_tf32(v.w);
    sts128(base + i, v);
  }
}

template <int BN, int MT>
__global__ void __launch_bounds__(TC_THREADS, tc_min_ctas(BN, MT))
conv_tc_kernel(const __grid_constant__ AMaps tm_as, const __grid_constant__ CUtensorMap tm_b, const TcParams p,
               const __grid_constant__ AMaps tm_e, const __grid_constant__ AMaps tm_o) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve: [stages][MT x A 16KB][B BN*128B] | barriers (256 B) | with ep_tma: the bias of the CTA's BN columns
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int b_bytes = BN * TC_BK * 4;
  constexpr int a_bytes = MT * TC_A_BYTES;
  constexpr int stage_bytes = a_bytes + b_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + p.stages * stage_bytes);
  uint64_t* empty_bar = full_bar + p.stages;
  float* s_bias = reinterpret_cast<float*>(smem + p.stages * stage_bytes + 256);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tap0 = p.ph_tap0[blockIdx.z];
  const int num_kb = (p.ph_tap0[blockIdx.z + 1] - tap0) * p.kchunks;

  // this CTA's pixel tiles: [tile0, tile0 + nt_here).  They all multiply the same weight tile, which is therefore
  // fetched from L2 once per k-block for MT*128 pixels.
  const int tile0 = blockIdx.x * MT;
  const int nt_here = max(0, min(MT, p.tiles_total - tile0));
  const int nb0 = blockIdx.y * BN;          // first output channel of this CTA

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);            // one arrive per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == TC_CWARPS) {
    // ===== TMA producer =====
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_as.m[0]) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_b) : "memory");
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        const int tl = kb / p.kchunks, kc = kb - tl * p.kchunks, tap = tap0 + tl;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * stage_bytes;
        uint8_t* sb = sa + a_bytes;
        mbar_expect_tx(&full_bar[stage], (uint32_t)(nt_here * p.rows_used * TC_BK * 4 + b_bytes));
        int ow0, oh0, n0;
        for (int i = 0; i < nt_here; ++i) {
          tc_tile_origin(p, tile0 + i, ow0, oh0, n0);
          tma_load_4d(sa + i * TC_A_BYTES, &tm_as.m[p.amap[tap]], &full_bar[stage], kc * TC_BK, ow0 + p.off_w[tap],
                      oh0 + p.off_h[tap], n0);
        }
        tc_tile_origin(p, tile0, ow0, oh0, n0);   // batched GEMM: all tiles of a CTA lie in one image (host guarantees)
        tma_load_3d(sb, &tm_b, &full_bar[stage], kc * TC_BK, nb0, p.wtap[tap] + n0 * p.wimg_stride);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      if (p.ep_tma) {
        // the epilogue's slots, one per 32-column chunk of the CTA's tiles: the first one is handed over while the
        // consumers still run the last stages - 1 k-blocks.  With a residual / mask the chunk of it is loaded into the
        // slot; box rows past the grid, or past the phase's own extent (the map of each phase has that extent), are
        // zero-filled and count in the bytes.
        const CUtensorMap* em = &tm_e.m[blockIdx.z];
        for (int t = 0; t < nt_here; ++t) {
          int ow0, oh0, n0;
          tc_tile_origin(p, tile0 + t, ow0, oh0, n0);
          for (int cc = 0; cc < BN / 32; ++cc) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            if (p.ep_smem) {
              mbar_expect_tx(&full_bar[stage], (uint32_t)(p.rows_used * TC_BK * 4));
              tma_load_4d(smem + stage * stage_bytes, em, &full_bar[stage], nb0 + cc * 32, ow0, oh0, n0);
            } else {
              mbar_arrive(&full_bar[stage]);
            }
            if (++stage == p.stages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ===== consumer warpgroups =====
    const int wg = warp >> 2;
    const int q = threadIdx.x & 127;
    if (p.ep_tma && p.bias)
      for (int i = threadIdx.x; i < BN; i += 32 * TC_CWARPS) s_bias[i] = nb0 + i < p.cout ? p.bias[nb0 + i] : 0.f;
    float acc[MT][BN / 2];
#pragma unroll
    for (int t = 0; t < MT; ++t)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[t][i] = 0.f;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(smem + stage * stage_bytes) + wg * TC_WG_A_BYTES;
      const uint32_t b_addr = smem_u32(smem + stage * stage_bytes) + a_bytes;
      if (p.round_a) {
        for (int tl = 0; tl < nt_here; ++tl) tc_round_smem(a_addr + tl * TC_A_BYTES, TC_WG_A_BYTES, q, 128);
        fence_proxy_async();
        named_bar(1 + wg, 128);
      }
#pragma unroll
      for (int t = 0; t < MT; ++t)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc_fence(acc[t][i]);
      wgmma_fence();
      // every one of the MT tiles is multiplied (a tile past the grid's end holds stale rows that are never stored): one
      // unconditional chain of MMAs
#pragma unroll
      for (int t = 0; t < MT; ++t) {
#pragma unroll
        for (int k = 0; k < TC_BK / 8; ++k)     // K = 8 for tf32: 32 B per step inside the 128 B swizzle row
          wgmma_tf32<BN>(acc[t], make_desc(a_addr + t * TC_A_BYTES + k * 32), make_desc(b_addr + k * 32));
      }
      wgmma_commit();
      wgmma_wait<1>();                               // the previous k-block's MMAs have retired: free its stage
#pragma unroll
      for (int t = 0; t < MT; ++t)
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc_fence(acc[t][i]);
      if (prev >= 0 && q == 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == p.stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (p.ep_tma) {
      // the last k-block's stage goes back to the producer for the epilogue's chunks
      if (prev >= 0 && q == 0) mbar_arrive(&empty_bar[prev]);
      named_bar(3, 32 * TC_CWARPS);              // s_bias is written
      int chunk = 0;
#pragma unroll
      for (int t = 0; t < MT; ++t) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc_fence(acc[t][i]);
        if (t < nt_here)
          tile_epilogue_smem<BN>(p, &tm_o.m[blockIdx.z], acc[t], tile0 + t, nb0, wg, warp, lane, smem, stage_bytes,
                                 full_bar, empty_bar, stage, phase, chunk, nt_here * (BN / 32), smem_u32(s_bias));
      }
      if (threadIdx.x == 0) bulk_wait_read<0>();   // the ring stays allocated until the last store has read it
    } else {
#pragma unroll
      for (int t = 0; t < MT; ++t) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc_fence(acc[t][i]);
        if (t < nt_here) tile_epilogue<BN>(p, acc[t], tile0 + t, nb0, wg, warp, lane, p.ph_base[blockIdx.z]);
      }
    }
  }
}

// ---- halo variant ------------------------------------------------------------------------------------------------
// 3x3 stride-1 convolutions whose activation operand still has to be rounded: per 32-channel k-block a CTA would pull
// 16 KB of activations per pixel tile for every one of the nine taps although the nine boxes overlap almost completely.
// Here the three taps of one kernel COLUMN share a single TMA box of bh + 2 image rows; the vertical shift of a tap is a
// descriptor start-address offset of bw pixel rows (a multiple of 1024 B, so the 128B-swizzle phase is unchanged).  The
// activation operand is fetched 3 x (bh+2)/bh times per chunk instead of 9 x, which also cuts the in-smem rounding work
// by the same factor.  Activations and weights run in two rings of their own (a halo box lives for three k-blocks).
template <int BN, int MT>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_tc_halo_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b, const TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int b_bytes = BN * TC_BK * 4;
  const int a_stage = MT * p.a_halo_bytes;
  uint8_t* smem_b = smem + p.sa_stages * a_stage;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem_b + p.sb_stages * b_bytes);
  uint64_t* a_empty = a_full + p.sa_stages;
  uint64_t* b_full = a_empty + p.sa_stages;
  uint64_t* b_empty = b_full + p.sb_stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile0 = blockIdx.x * MT;
  const int nt_here = min(MT, p.tiles_total - tile0);
  const int nb0 = blockIdx.y * BN;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.sa_stages; ++s) {
      mbar_init(&a_full[s], 1);
      mbar_init(&a_empty[s], 2);
    }
    for (int s = 0; s < p.sb_stages; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == TC_CWARPS) {
    // ===== TMA producer: per (channel chunk, tap column) one halo box per tile, then the hnv weight tiles =====
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_a) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_b) : "memory");
      int sa = 0, sb = 0;
      uint32_t pa = 0, pb = 0;
      for (int kc = 0; kc < p.kchunks; ++kc) {
        for (int g = 0; g < p.hg; ++g) {
          mbar_wait(&a_empty[sa], pa ^ 1);
          mbar_expect_tx(&a_full[sa], (uint32_t)(nt_here * p.a_box_bytes));
          for (int i = 0; i < nt_here; ++i) {
            int ow0, oh0, n0;
            tc_tile_origin(p, tile0 + i, ow0, oh0, n0);
            tma_load_4d(smem + sa * a_stage + i * p.a_halo_bytes, &tm_a, &a_full[sa], kc * TC_BK, ow0 + p.h_off_w[g],
                        oh0 + p.h_off_h0[g], n0);
          }
          if (++sa == p.sa_stages) { sa = 0; pa ^= 1; }
          for (int t = 0; t < p.hnv; ++t) {
            mbar_wait(&b_empty[sb], pb ^ 1);
            mbar_expect_tx(&b_full[sb], (uint32_t)b_bytes);
            tma_load_3d(smem_b + sb * b_bytes, &tm_b, &b_full[sb], kc * TC_BK, nb0, p.h_wtap[g][t]);
            if (++sb == p.sb_stages) { sb = 0; pb ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ===== consumer warpgroups =====
  const int wg = warp >> 2;
  float acc[MT][BN / 2];
#pragma unroll
  for (int t = 0; t < MT; ++t)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[t][i] = 0.f;
  const uint32_t tap_shift = (uint32_t)(p.bw * 128);          // one image row of the box = bw pixel rows of 128 B
  int sa = 0, sb = 0, prev_a = -1, prev_b = -1;
  uint32_t pa = 0, pb = 0;
  for (int kc = 0; kc < p.kchunks; ++kc) {
    for (int g = 0; g < p.hg; ++g) {
      mbar_wait(&a_full[sa], pa);
      const uint32_t a_addr = smem_u32(smem + sa * a_stage);
      if (p.round_a) {          // the box rows are shared by both warpgroups: round it together, then sync the two
        for (int tl = 0; tl < nt_here; ++tl) tc_round_smem(a_addr + tl * p.a_halo_bytes, p.a_box_bytes, threadIdx.x, 256);
        fence_proxy_async();
        named_bar(1, 256);
      }
      for (int t = 0; t < p.hnv; ++t) {
        mbar_wait(&b_full[sb], pb);
        const uint32_t b_addr = smem_u32(smem_b + sb * b_bytes);
#pragma unroll
        for (int u = 0; u < MT; ++u)
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc_fence(acc[u][i]);
        wgmma_fence();
#pragma unroll
        for (int u = 0; u < MT; ++u) {
#pragma unroll
          for (int k = 0; k < TC_BK / 8; ++k)
            wgmma_tf32<BN>(acc[u], make_desc(a_addr + u * p.a_halo_bytes + t * tap_shift + wg * TC_WG_A_BYTES + k * 32),
                           make_desc(b_addr + k * 32));
        }
        wgmma_commit();
        wgmma_wait<1>();
#pragma unroll
        for (int u = 0; u < MT; ++u)
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc_fence(acc[u][i]);
        // the previous group of MMAs has retired: release its weight tile (and its halo box after a column's last tap)
        if ((threadIdx.x & 127) == 0) {
          if (prev_b >= 0) mbar_arrive(&b_empty[prev_b]);
          if (prev_a >= 0) mbar_arrive(&a_empty[prev_a]);
        }
        prev_b = sb;
        prev_a = (t == p.hnv - 1) ? sa : -1;
        if (++sb == p.sb_stages) { sb = 0; pb ^= 1; }
      }
      if (++sa == p.sa_stages) { sa = 0; pa ^= 1; }
    }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int t = 0; t < MT; ++t) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc_fence(acc[t][i]);
    if (t < nt_here) tile_epilogue<BN>(p, acc[t], tile0 + t, nb0, wg, warp, lane, p.base);
  }
}

// dst[tap][r][k] (r < rows_pad) = rna_tf32(src[tap][k][r]) (transpose) or rna_tf32(src[tap][r][k]); rows >= `rows` are 0
__global__ void wprep_kernel(float* __restrict__ dst, const float* __restrict__ src, int taps, int rows, int rows_pad,
                             int kdim, int kdim_pad, int transpose) {
  long long tot = (long long)taps * rows_pad * kdim_pad;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (long long)gridDim.x * blockDim.x) {
    int k = (int)(i % kdim_pad);
    long long t = i / kdim_pad;
    int r = (int)(t % rows_pad);
    int tap = (int)(t / rows_pad);
    float v = 0.f;
    if (r < rows && k < kdim)
      v = transpose ? src[((long long)tap * kdim + k) * rows + r] : src[((long long)tap * rows + r) * kdim + k];
    dst[i] = rna_tf32(v);
  }
}

// 128-pixel tile = bni images x bh rows x bw columns (bw*bh*bni <= 128).  Any grid size is accepted: border tiles hang
// over (TMA zero-fills, the epilogue masks), e.g. Inception's 35x35 maps use 35x3 boxes (105 of 128 MMA rows).
inline void tc_geometry(int n, int h, int w, int* bw, int* bh, int* bni, int* tw, int* th, int* tn) {
  int parts = (w + 127) / 128;
  *bw = (w + parts - 1) / parts;
  *tw = (w + *bw - 1) / *bw;
  *bh = 128 / *bw; if (*bh > h) *bh = h; if (*bh < 1) *bh = 1;
  *th = (h + *bh - 1) / *bh;
  *bni = (*bh == h) ? 128 / (*bw * *bh) : 1;
  if (*bni < 1) *bni = 1;
  if (*bni > n) *bni = n;
  *tn = (n + *bni - 1) / *bni;
}

inline int tc_pick_bn(int ncols_pad) {     // largest wgmma N <= 256 (multiple of 32) that divides the padded column count
  if (ncols_pad <= 256) return ncols_pad;
  for (int b = 256; b >= 32; b -= 32)
    if (ncols_pad % b == 0) return b;
  return 0;
}

// Few pixel tiles (8x8 / 17x17 Inception stages at batch 64, the 4x4 GAN stages): the widest column tile would leave SMs
// idle, so the columns are split further (>= 64) until there is at least one CTA per SM.  The K order is unchanged, so
// the result is bit-identical to the wide tile's.
inline int tc_pick_bn_occupancy(int ncols_pad, long long tiles_m, int sms) {
  int best = tc_pick_bn(ncols_pad);
  if (best == 0 || tiles_m * (ncols_pad / best) >= sms) return best;
  int pick = best;
  for (int b = best - 32; b >= 64; b -= 32) {
    if (ncols_pad % b) continue;
    pick = b;
    if (tiles_m * (ncols_pad / b) >= sms) break;
  }
  return pick;
}

// Column tile of the per-tap kernel.  A 256-wide tile holds 128 fp32 accumulators per consumer thread, so only one CTA
// fits on an SM and the tensor cores idle through every epilogue store and pipeline fill.  Two 128-wide CTAs share an SM
// and one's epilogue overlaps the other's main loop; that is worth more than the doubled activation bytes per MMA while
// the K loop is short (on H100: the generator's 3x3 256->256 convolutions at 16x16 and 32x32, batch 256, 72 k-blocks,
// run 15-20 % faster) but not once it is long (BigGAN-128's 768-column convolutions at 16x16, 216 k-blocks, 35 % slower).
// So the tile is halved when there are at least TC_NARROW_WAVES waves of 256-wide CTAs (pixel tiles x column tiles x
// phases) and at most TC_NARROW_MAX_KB k-blocks (taps of the longest phase x 32-channel chunks) per CTA.  The K order is
// unchanged, so the result is bit-identical to the wide tile's.
constexpr int TC_NARROW_WAVES = 2;
constexpr int TC_NARROW_MAX_KB = 96;

inline int tc_pick_bn_per_tap(int ncols_pad, long long tiles_m, const TcParams& p, int sms) {
  const int bn = tc_pick_bn_occupancy(ncols_pad, tiles_m, sms);
  int kb = 0;
  for (int i = 0; i < p.nphases; ++i) {
    const int k = (p.ph_tap0[i + 1] - p.ph_tap0[i]) * p.kchunks;
    if (k > kb) kb = k;
  }
  if (bn == 256 && tiles_m * (ncols_pad / 256) * p.nphases >= (long long)TC_NARROW_WAVES * sms && kb <= TC_NARROW_MAX_KB)
    return 128;
  return bn;
}


// every output row of the launch starts at an even element offset and the column count is even: float2 epilogue
inline int tc_vec2(const TcParams& p) {
  long long odd = p.cout | p.s_n | p.s_h | p.s_w | p.base;
  for (int i = 0; i < p.nphases; ++i) odd |= p.ph_base[i];
  return (odd & 1) ? 0 : 1;
}

// The per-tap kernel stages its epilogue through the stage ring and stores the tiles by TMA (tile_epilogue_smem) when the
// float2 epilogue applies, the launch has at most one of residual / mask, and TMA can address the output (and that
// operand) in the output's geometry: bases, every phase's first element and the pixel strides 16-byte aligned.  Any
// other launch (a channel slice at an unaligned offset or width, residual and mask together) keeps tile_epilogue.
inline bool tc_ep_tma_ok(const TcParams& p, const TcConv& c) {
  const float* e = c.residual ? c.residual : c.mask;
  if (!p.vec2 || (c.residual && c.mask) || ((reinterpret_cast<uintptr_t>(c.out) | reinterpret_cast<uintptr_t>(e)) & 15))
    return false;
  long long a = p.s_n | p.s_h | p.s_w;
  for (int i = 0; i < p.nphases; ++i) a |= p.ph_base[i];
  return (a & 3) == 0;
}

// Kernel parameters of conv_tc_kernel, within the 4 KB a launch may pass: three AMaps (activation views, residual /
// mask views, output views) of 4 x 128 B, one 128 B weight map and TcParams, plus at most 2 x 63 B of padding in front
// of the 64-byte aligned maps after TcParams.
static_assert(3 * sizeof(AMaps) + sizeof(CUtensorMap) + sizeof(TcParams) + 2 * 63 <= 4096, "conv_tc_kernel parameters");

// Weights -> TF32-rounded (nearest) K-major [taps_total][ncols_pad][kdim_pad] in the context workspace
int prep_weights(cgan_ctx* ctx, const TcConv& c, int kdim_pad, int ncols_pad, float** out) {
  void* ws = nullptr;
  int rc = cgan_ws(ctx, (size_t)c.taps_total * ncols_pad * kdim_pad * sizeof(float), &ws);
  if (rc) return rc;
  float* wt = reinterpret_cast<float*>(ws);
  long long tot = (long long)c.taps_total * ncols_pad * kdim_pad;
  long long blocks = (tot + 255) / 256, cap = (long long)ctx->num_sms * 8;
  wprep_kernel<<<(int)(blocks > cap ? cap : blocks), 256, 0, ctx->stream>>>(wt, c.wsrc, c.taps_total, c.ncols, ncols_pad, c.a.ch,
                                                                             kdim_pad, c.transpose_w);
  CGAN_LAUNCHED(ctx);
  *out = wt;
  return CGAN_OK;
}

// 3-D map {k, column, tap} of the prepared weights, 128B-swizzled boxes of 32 channels x bn columns of one tap
bool make_weight_map(CUtensorMap* tm, float* wt, int kdim_pad, int ncols_pad, int taps_total, int bn) {
  cuuint64_t dims[3] = {(cuuint64_t)kdim_pad, (cuuint64_t)ncols_pad, (cuuint64_t)taps_total};
  cuuint64_t strides[2] = {(cuuint64_t)kdim_pad * 4, (cuuint64_t)ncols_pad * kdim_pad * 4};
  cuuint32_t box[3] = {TC_BK, (cuuint32_t)bn, 1};
  cuuint32_t es[3] = {1, 1, 1};
  return get_encode()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, wt, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// CTAs of `kernel` that fit on one SM at `smem` bytes of dynamic shared memory (CGAN_OPT_LAST_TC_CTAS_PER_SM)
template <typename Kernel>
int tc_ctas_per_sm(Kernel kernel, size_t smem) {
  int blocks = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kernel, TC_THREADS, smem) != cudaSuccess) blocks = 0;
  return blocks;
}

// halo: the halo kernel, reading the activation box through as.m[0]
template <int BN, int MT>
int tc_launch_t(cgan_ctx* ctx, bool halo, dim3 grid, size_t smem, const AMaps& as, const CUtensorMap& b, const TcParams& p,
                const AMaps& es, const AMaps& os) {
  static bool attr_set[2] = {false, false};
  if (halo) {
    if (!attr_set[1]) {
      CGAN_CUDA(ctx, cudaFuncSetAttribute(conv_tc_halo_kernel<BN, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      attr_set[1] = true;
    }
    ctx->last_tc_ctas_per_sm = tc_ctas_per_sm(conv_tc_halo_kernel<BN, MT>, smem);
    conv_tc_halo_kernel<BN, MT><<<grid, TC_THREADS, smem, ctx->stream>>>(as.m[0], b, p);
  } else {
    if (!attr_set[0]) {
      CGAN_CUDA(ctx, cudaFuncSetAttribute(conv_tc_kernel<BN, MT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      attr_set[0] = true;
    }
    ctx->last_tc_ctas_per_sm = tc_ctas_per_sm(conv_tc_kernel<BN, MT>, smem);
    conv_tc_kernel<BN, MT><<<grid, TC_THREADS, smem, ctx->stream>>>(as, b, p, es, os);
  }
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

// the accumulator fragment is sized at compile time: one instantiation per (bn, mt), mt * bn <= TC_ACC_COLS.  es: the
// residual / mask views of a launch with ep_smem, os: the output views of a launch with ep_tma (unused otherwise)
int tc_launch(cgan_ctx* ctx, bool halo, dim3 grid, size_t smem, const AMaps& as, const CUtensorMap& b, const TcParams& p,
              const AMaps& es, const AMaps& os) {
  ctx->last_tc_bn = p.bn; ctx->last_tc_mt = p.mt; ctx->last_tc_halo = halo ? 1 : 0; ctx->last_tc_ep_smem = p.ep_smem;
  ctx->last_tc_tma_store = p.ep_tma;
#define TC_CASE(BN, MT) \
  if (p.bn == BN && p.mt == MT) return tc_launch_t<BN, MT>(ctx, halo, grid, smem, as, b, p, es, os);
  TC_CASE(32, 1) TC_CASE(64, 1) TC_CASE(96, 1) TC_CASE(128, 1) TC_CASE(160, 1) TC_CASE(192, 1) TC_CASE(224, 1)
  TC_CASE(256, 1) TC_CASE(32, 2) TC_CASE(64, 2) TC_CASE(96, 2) TC_CASE(128, 2)
#undef TC_CASE
  return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: no kernel for this column tile / pixel-tile count%s", "cgan_conv_tc");
}

}  // namespace

bool cgan_tc_shape_ok(int n, int h, int w, int kdim, int ncols) {
  if (n < 1 || h < 1 || w < 1 || ncols < 1) return false;
  if (kdim < 8 || kdim % 4 != 0) return false;           // TMA needs 16-byte pixel strides; K is zero-padded to 32
  if (ncols > 256 && ncols % 32 != 0) return false;      // small column counts are zero-padded to a multiple of 32
  int bn = tc_pick_bn((ncols + 31) / 32 * 32);
  return bn != 0 && bn % 32 == 0;
}

int cgan_conv_tc(cgan_ctx* ctx, const TcConv& c) {
  if (!get_encode()) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: cuTensorMapEncodeTiled unavailable%s", "cgan_conv_tc");
  const ConvTaps& tp = c.taps;
  if (tp.ntaps > TC_MAX_TAPS || c.a.nviews > 4) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: too many taps/views%s", "cgan_conv_tc");
  const int n = c.a.n, h = c.a.h, w = c.a.w, kdim = c.a.ch, gh = c.gh, gw = c.gw, ntaps = tp.ntaps;
  TcParams p;
  memset(&p, 0, sizeof(p));
  p.ntaps = ntaps;
  const int kdim_pad = (kdim + TC_BK - 1) / TC_BK * TC_BK;
  p.kchunks = kdim_pad / TC_BK;
  for (int i = 0; i < ntaps; ++i) {
    p.off_h[i] = tp.off_h[i]; p.off_w[i] = tp.off_w[i]; p.wtap[i] = tp.wtap[i]; p.amap[i] = tp.view[i];
  }
  int tiles_n;
  // the pixel grid that is tiled (gh x gw: the OUTPUT extent) may differ from the extent of the input views (h x w):
  // VALID convolutions shrink it, their taps only carry non-negative offsets
  tc_geometry(n, gh, gw, &p.bw, &p.bh, &p.bni, &p.tiles_w, &p.tiles_h, &tiles_n);
  p.rows_used = p.bw * p.bh * p.bni;
  p.img_n = n;
  p.relu = c.relu;
  p.round_a = c.a.tf32 ? 0 : 1;
  p.round_out = c.round_out; p.residual = c.residual; p.mask = c.mask; p.mask_leak = c.mask_leak;
  p.mask_thr = relu_gate_threshold(c.mask_leak);
  p.nphases = 1;
  p.ph_tap0[0] = 0; p.ph_tap0[1] = ntaps;
  p.ph_base[0] = c.base;
  for (int i = 0; i < 4; ++i) {
    p.ph_h[i] = c.ph_h[i] ? c.ph_h[i] : gh;
    p.ph_w[i] = c.ph_w[i] ? c.ph_w[i] : gw;
  }
  if (tp.nphases > 1) {
    if (tp.nphases > 4) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: more than four phases%s", "cgan_conv_tc");
    p.nphases = tp.nphases;
    for (int i = 0; i <= tp.nphases; ++i) p.ph_tap0[i] = tp.ph_tap0[i];
    for (int i = 0; i < tp.nphases; ++i) p.ph_base[i] = c.ph_base[i];
  }
  p.wimg_stride = c.wimg_stride;
  if (c.wimg_stride != 0 && p.bni != 1)
    return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: batched GEMM needs >= 128 rows per matrix%s", "cgan_conv_tc");
  const int ncols_pad = (c.ncols + 31) / 32 * 32;
  p.bn = tc_pick_bn_per_tap(ncols_pad, (long long)p.tiles_w * p.tiles_h * tiles_n, p, ctx->num_sms);
  p.cout = c.ncols;
  p.s_n = c.s_n; p.s_h = c.s_h; p.s_w = c.s_w; p.base = c.base;
  p.out = c.out;
  p.bias = c.bias;

  float* wt = nullptr;
  int rc = prep_weights(ctx, c, kdim_pad, ncols_pad, &wt);
  if (rc) return rc;

  // ---- halo variant: three taps of a kernel column share one (bh+2)-row activation box --------------------------------
  // Used where the activation operand still has to be rounded in shared memory (the halo box cuts that work 9 -> 3 x
  // (bh+2)/bh per chunk); a pre-rounded operand streams through the per-tap kernel.  CGAN_OPT_TC_HALO = 2 forces it
  // everywhere (tests).
  const bool halo_wanted = ctx->tc_halo == 2 || (ctx->tc_halo == 1 && p.round_a && ncols_pad >= 256);
  if (halo_wanted && p.nphases == 1 && c.a.nviews == 1 && c.wimg_stride == 0 && ntaps == 9 && gh == h && gw == w) {
    int hbw = 0, hbh = 0;
    if (w % 32 == 0) { hbw = 32; hbh = 4; } else if (w == 16) { hbw = 16; hbh = 8; }
    // group the taps by horizontal offset; each group must be three vertically consecutive taps
    int gw_off[4], gh0[4], gcnt[4] = {0, 0, 0, 0}, gtap[4][4], ng = 0;
    bool ok = hbw != 0 && h % hbh == 0 && h >= hbh;
    for (int i = 0; ok && i < ntaps; ++i) {
      int g = -1;
      for (int j = 0; j < ng; ++j)
        if (gw_off[j] == tp.off_w[i]) g = j;
      if (g < 0) {
        if (ng == 3) { ok = false; break; }
        g = ng++; gw_off[g] = tp.off_w[i]; gh0[g] = tp.off_h[i];
      }
      if (gcnt[g] == 3) { ok = false; break; }
      if (tp.off_h[i] < gh0[g]) gh0[g] = tp.off_h[i];
      gtap[g][gcnt[g]++] = i;
    }
    ok = ok && ng == 3;
    for (int g = 0; ok && g < ng; ++g) {
      if (gcnt[g] != 3) { ok = false; break; }
      int ordered[3] = {-1, -1, -1};
      for (int j = 0; j < 3; ++j) {
        int dh = tp.off_h[gtap[g][j]] - gh0[g];
        if (dh < 0 || dh > 2 || ordered[dh] >= 0) { ok = false; break; }
        ordered[dh] = tp.wtap[gtap[g][j]];
      }
      for (int j = 0; ok && j < 3; ++j) p.h_wtap[g][j] = ordered[j];
      p.h_off_w[g] = gw_off[g]; p.h_off_h0[g] = gh0[g];
    }
    if (ok) {
      p.hg = 3; p.hnv = 3;
      p.bw = hbw; p.bh = hbh; p.bni = 1;
      p.tiles_w = w / hbw; p.tiles_h = h / hbh;
      const long long tiles_total = (long long)p.tiles_w * p.tiles_h * n;
      p.rows_used = 128;
      p.bn = tc_pick_bn_occupancy(ncols_pad, tiles_total, ctx->num_sms);
      const int ncol_tiles = ncols_pad / p.bn;
      p.a_box_bytes = (hbh + 2) * hbw * 128;
      p.a_halo_bytes = (p.a_box_bytes + 1023) / 1024 * 1024;
      const int b_bytes = p.bn * TC_BK * 4;
      // pixel tiles per CTA (they share every weight tile): as many as the accumulator registers hold (mt x bn <= 256),
      // while two waves of CTAs remain and the weight ring keeps >= 4 stages.  The activation ring has two stages, each
      // good for three k-blocks.
      const int budget = 227 * 1024 - 1024 - 512;
      const int mt_cap = ctx->tc_mt_max >= 2 ? 2 : 1;
      p.sa_stages = 2;
      p.mt = 1;
      for (int m = mt_cap; m >= 2; --m) {
        if (m * p.bn > TC_ACC_COLS || tiles_total * ncol_tiles < 2ll * m * ctx->num_sms) continue;
        if ((budget - p.sa_stages * m * p.a_halo_bytes) / b_bytes < 4) continue;
        p.mt = m;
        break;
      }
      p.sb_stages = (budget - p.sa_stages * p.mt * p.a_halo_bytes) / b_bytes;
      if (p.sb_stages > 8) p.sb_stages = 8;
      ok = p.sb_stages >= 2;
      if (ok) {
        p.tiles_total = (int)tiles_total;
        AMaps tm_a;
        CUtensorMap tm_b;
        memset(&tm_a, 0, sizeof(tm_a));
        if (!make_act_map(&tm_a.m[0], c.a.in + c.a.view_off[0], kdim, w, h, n, c.a.sw, c.a.sh, c.a.sn, hbw, hbh + 2, 1))
          return cgan_fail(ctx, CGAN_ERR_CUDA, "%s: cuTensorMapEncodeTiled(A halo) failed%s", "cgan_conv_tc");
        if (!make_weight_map(&tm_b, wt, kdim_pad, ncols_pad, c.taps_total, p.bn))
          return cgan_fail(ctx, CGAN_ERR_CUDA, "%s: cuTensorMapEncodeTiled(B) failed%s", "cgan_conv_tc");
        p.vec2 = tc_vec2(p);
        size_t smem = (size_t)p.sa_stages * p.mt * p.a_halo_bytes + (size_t)p.sb_stages * b_bytes + 1024 + 512;
        dim3 grid((unsigned)((tiles_total + p.mt - 1) / p.mt), (unsigned)ncol_tiles);
        return tc_launch(ctx, true, grid, smem, tm_a, tm_b, p, tm_a, tm_a);
      }
    }
    // not eligible after all: restore the standard geometry
    tc_geometry(n, gh, gw, &p.bw, &p.bh, &p.bni, &p.tiles_w, &p.tiles_h, &tiles_n);
    p.rows_used = p.bw * p.bh * p.bni;
    p.bn = tc_pick_bn_per_tap(ncols_pad, (long long)p.tiles_w * p.tiles_h * tiles_n, p, ctx->num_sms);
    p.hg = p.hnv = 0;
  }

  AMaps tm_as;
  CUtensorMap tm_b;
  memset(&tm_as, 0, sizeof(tm_as));
  for (int v = 0; v < 4; ++v)
    if (!make_view_map(&tm_as.m[v], c.a, v, p.bw, p.bh, p.bni))
      return cgan_fail(ctx, CGAN_ERR_CUDA, "%s: cuTensorMapEncodeTiled(A) failed%s", "cgan_conv_tc");
  if (!make_weight_map(&tm_b, wt, kdim_pad, ncols_pad, c.taps_total, p.bn))
    return cgan_fail(ctx, CGAN_ERR_CUDA, "%s: cuTensorMapEncodeTiled(B) failed%s", "cgan_conv_tc");

  // Pixel tiles per CTA: with mt = 2 the weight tile is fetched once for 256 pixels, which cuts the L2->SM bytes per MMA
  // by a third; only when enough CTAs remain to fill the machine.  Up to ~110 KB of smem per CTA when mt x bn <= 128, so
  // that two CTAs share an SM (tc_min_ctas keeps the registers within that too) and one's epilogue overlaps the other's
  // main loop.  That overlap is worth more than the bytes: on H100 the 3x3 128->128 conv at 32x32, batch 512, takes
  // 0.74 ms at bn = 128, mt = 1 (two CTAs per SM) against 1.39 ms at mt = 2 (one CTA per SM).  So mt = 2 only where two
  // such CTAs still share an SM: bn <= 64.
  const long long tiles_total = (long long)p.tiles_w * p.tiles_h * tiles_n;
  const int ncol_tiles = ncols_pad / p.bn;
  p.tiles_total = (int)tiles_total;
  p.mt = 1;
  if (ctx->tc_mt_max >= 2 && 2 * p.bn <= 128 && tiles_total * ncol_tiles * p.nphases >= 4ll * ctx->num_sms &&
      (c.wimg_stride == 0 || (p.tiles_w * p.tiles_h) % 2 == 0))
    p.mt = 2;
  const bool two_ctas = p.mt * p.bn <= 128;
  const size_t stage_bytes = (size_t)p.mt * TC_A_BYTES + (size_t)p.bn * TC_BK * 4;
  p.stages = (int)(((two_ctas ? 110 : 220) * 1024) / stage_bytes);
  if (p.stages > TC_MAX_STAGES) p.stages = TC_MAX_STAGES;
  if (p.stages < 2) p.stages = 2;
  p.vec2 = tc_vec2(p);
  AMaps tm_e, tm_o;
  memset(&tm_e, 0, sizeof(tm_e));
  memset(&tm_o, 0, sizeof(tm_o));
  p.ep_tma = tc_ep_tma_ok(p, c) ? 1 : 0;
  p.ep_smem = p.ep_tma && (c.residual || c.mask) ? 1 : 0;
  for (int v = 0; p.ep_tma && v < p.nphases; ++v) {
    if (!make_act_map(&tm_o.m[v], c.out + p.ph_base[v], c.ncols, p.ph_w[v], p.ph_h[v], n, p.s_w, p.s_h, p.s_n, p.bw, p.bh,
                      p.bni))
      return cgan_fail(ctx, CGAN_ERR_CUDA, "%s: cuTensorMapEncodeTiled(output) failed%s", "cgan_conv_tc");
    if (p.ep_smem && !make_act_map(&tm_e.m[v], (c.residual ? c.residual : c.mask) + p.ph_base[v], c.ncols, p.ph_w[v],
                                   p.ph_h[v], n, p.s_w, p.s_h, p.s_n, p.bw, p.bh, p.bni))
      return cgan_fail(ctx, CGAN_ERR_CUDA, "%s: cuTensorMapEncodeTiled(residual / mask) failed%s", "cgan_conv_tc");
  }
  size_t smem = (size_t)p.stages * stage_bytes + 1024 /*align*/ + 256 /*barriers*/ + (p.ep_tma ? p.bn * 4 : 0) /*bias*/;
  dim3 grid((unsigned)((tiles_total + p.mt - 1) / p.mt), (unsigned)ncol_tiles, (unsigned)p.nphases);
  return tc_launch(ctx, false, grid, smem, tm_as, tm_b, p, tm_e, tm_o);
}
