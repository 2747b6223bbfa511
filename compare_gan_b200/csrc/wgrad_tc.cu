// Warpgroup-MMA (wgmma, sm_90a) filter-gradient kernel (math_mode 1):
//
//   dW[tap][ci][co] = sum_pixels  X[pixel + off(tap)][ci] * dY[pixel][co]
//
// A GEMM whose reduction dimension is the PIXEL index, so both operands are "MN-major" as they lie in HBM (NHWC:
// channels contiguous): D[ci, co] += A[ci, pix] * B[pix, co].  Per k-block of 32 pixels, TMA brings
//   * 4 boxes  [32 pixels x 32 ci]  of X per (tap, ci-tile) unit (shifted by the tap offset; SAME padding = TMA zero
//     fill), 128B-swizzled, and
//   * N/32 boxes [32 pixels x 32 co] of dY, unswizzled,
// each box = 32 rows x 128 B.  wgmma takes 32-bit shared-memory operands only K-major, so X goes to the MMAs from
// registers: each consumer thread loads its m64k8 A fragments (two adjacent ci, one pixel per LDS.64) straight out of the
// TMA stage, conflict-free thanks to the swizzle, and rounds them to nearest TF32 there.  Only dY is transposed by the
// two consumer warpgroups into a 128B-swizzled K-major tile (one 128-byte row of 32 pixels per co), rounded on the way,
// into one of two buffers; the TMA stage is released once its fragments are loaded and its dY transposed.  Four wgmma
// m64nNk8 per unit and warpgroup (K = 8 pixels) consume a k-block, in two commit groups: the fragments of one group are
// loaded while the other's MMAs run; warpgroup g owns ci rows 64g..64g+63 of each unit.
// Per k-block of wgrad_tc_kernel<128, 2> that is 48 KB of TMA writes, 32 KB of fragment loads, 16 + 16 KB of dY
// transpose and 64 KB of wgmma B reads, 176 KB of shared-memory traffic where transposing X as well took 240 KB.
// The pixel range is split across CTAs (split-K); partial tiles go to a workspace and are summed in a fixed order
// (deterministic), replacing TF's Conv2DBackpropFilter.
// A conv over a zero-inserted 2x-upsampled input (resnet_ops.py:35-56) is handled through four strided TMA views of dY
// (one per sub-pixel phase); every tap belongs to exactly one phase.
// A grid whose width neither divides 32 nor is a multiple of it (the 48, 24, 12, 6 and 3 wide maps of a 48x48 network)
// takes a box of at most 32 pixels that may hang over the grid's edge (`box_any`): TMA zero-fills the overrun, a zero dY
// pixel adds nothing to dW, and the pixel rows the box leaves empty are zeroed once per CTA and never written again.
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int WG_MAX_STAGES = 4;
constexpr int WG_P = 32;                 // pixels per k-block
constexpr int WG_BOX = WG_P * 128;       // 4 KB: 32 pixel rows x 32 channels fp32
constexpr int WG_A_BYTES = 4 * WG_BOX;   // 128 input channels
constexpr int WG_CWARPS = 8;             // two consumer warpgroups
constexpr int WG_THREADS = 32 * WG_CWARPS + 128;   // + the producer warpgroup, one thread of which issues the TMA
constexpr int WG_MAX_TAPS = 16;
constexpr int WG_ACC_COLS = 256;         // mt x bn accumulator columns per CTA

struct WgParams {
  int ntaps;
  int off_h[WG_MAX_TAPS], off_w[WG_MAX_TAPS], amap[WG_MAX_TAPS], bmap[WG_MAX_TAPS], wtap[WG_MAX_TAPS];
  int bw, bh, bni, tiles_w, tiles_h;     // box geometry: bw x bh x bni <= 32 pixels, tiles of the grid per box
  int kblocks, kb_per_split;
  int ci_tiles, co_tiles, bn;
  int cin, cout, taps_total;
  int stages;                            // TMA ring depth
  int mt;                                // (tap, ci-tile) units per CTA that share one dY tile (mt accumulator tiles)
  int round_a, round_b;                  // round the X / dY tiles to nearest TF32 (operand not pre-rounded)
  float* partial;                        // [split][taps_total][cin][cout]
  int rows_used;                         // bw * bh * bni: pixel rows of a k-block the TMA box fills
};

struct BMaps { CUtensorMap m[4]; };

// [32 pixels][ROWS] (unswizzled boxes of 32 channels, box b at b * WG_BOX) -> K-major swizzled [ROWS][32 pixels].
// Consumer warp w (0..7) moves pixels 4w..4w+3 of every row, lane = channel within a box.  Each LDS.32 of a warp reads
// one 128-byte pixel row of a box (one wavefront); each STS.128 writes 4 pixels into rows 32b..32b+31 at 16-byte chunk
// (w ^ row) & 7, so every 8 consecutive rows take 8 distinct chunks and the warp's 512 bytes go out in 4 wavefronts,
// the minimum.  Loads are issued four boxes at a time ahead of their stores.
template <int ROWS>
__device__ __forceinline__ void wg_transpose(uint32_t dst, uint32_t src, bool round, int warp, int lane) {
  constexpr int NB = ROWS / 32;
#pragma unroll
  for (int b0 = 0; b0 < NB; b0 += 4) {
    float4 v[4];
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      if (b0 + b >= NB) break;
      const uint32_t s = src + (b0 + b) * WG_BOX + warp * 4 * 128 + lane * 4;
      v[b] = make_float4(lds32(s), lds32(s + 128), lds32(s + 256), lds32(s + 384));
    }
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      if (b0 + b >= NB) break;
      if (round) { v[b].x = rna_tf32(v[b].x); v[b].y = rna_tf32(v[b].y); v[b].z = rna_tf32(v[b].z); v[b].w = rna_tf32(v[b].w); }
      sts128(dst + sw128_offset((b0 + b) * 32 + lane, 4 * warp), v[b]);
    }
  }
}

// A operand of the m64nNk8 MMAs straight from the TMA stage.  The X boxes land 128B-swizzled: pixel row p at p * 128 B,
// its 16-byte chunk of channels 4c..4c+3 at chunk c ^ (p & 7).  Thread (warp, lane) feeds accumulator rows lane / 4 and
// lane / 4 + 8 of its warp's 16; they are the adjacent channels cib, cib + 1 of box 2 * wg + (warp & 3) / 2, so one LDS.64
// per pixel gives a[0], a[1] (pixel 8k + lane % 4) and one more a[2], a[3] (4 pixels on).  A half-warp's 16 lanes read
// 4 pixels x 4 channel pairs from two chunks 16 channels apart (cib / 4 differs in bit 2), which the swizzle spreads over
// all eight chunk positions: every LDS.64 takes the minimum two wavefronts.  Warp parity picks the other four chunks.
// keeps the compiler from sinking a fragment's rounding past wgmma.fence
__device__ __forceinline__ void frag_fence(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }

__device__ __forceinline__ int wg_a_channel(int warp, int lane) {
  const int r = lane >> 2;
  return 4 * (2 * (warp & 1) + (r >> 2) + 4 * ((r >> 1) & 1)) + 2 * (r & 1);
}

// the A fragments of GK consecutive k-steps, the first at src (a unit's boxes + k-step * 1024 B), rounded to nearest
// TF32 unless the operand is pre-rounded
template <int GK>
__device__ __forceinline__ void wg_load_a(uint32_t (&f)[GK][4], uint32_t src, uint32_t lo, uint32_t hi, bool round) {
#pragma unroll
  for (int e = 0; e < GK; ++e) {
    float2 a = lds64(src + e * 1024 + lo), b = lds64(src + e * 1024 + hi);
    if (round) { a.x = rna_tf32(a.x); a.y = rna_tf32(a.y); b.x = rna_tf32(b.x); b.y = rna_tf32(b.y); }
    f[e][0] = __float_as_uint(a.x); f[e][1] = __float_as_uint(a.y); f[e][2] = __float_as_uint(b.x); f[e][3] = __float_as_uint(b.y);
#pragma unroll
    for (int i = 0; i < 4; ++i) frag_fence(f[e][i]);    // rounded here, not next to the MMAs
  }
}

// PART: the box holds fewer than 32 pixels (box_any); box32's grids run the PART = false instantiations
template <int BN, int MT, bool PART>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ BMaps tm_x, const __grid_constant__ BMaps tm_dy, const WgParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int b_bytes = (BN / 32) * WG_BOX;
  constexpr int a_bytes = MT * WG_A_BYTES;
  constexpr int stage_bytes = a_bytes + b_bytes;
  // [stages] TMA ring | [2] transposed K-major dY tiles | barriers
  uint8_t* tbuf = smem + p.stages * stage_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(tbuf + 2 * b_bytes);
  uint64_t* empty_bar = full_bar + p.stages;
  uint64_t* buf_free = empty_bar + p.stages;    // [2] both warpgroups' MMAs reading dY buffer b have retired

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // work units (tap, ci tile); this CTA owns units [u0, u0 + nu) — they all contract against the same dY tile, which is
  // fetched from L2 once per k-block for all of them
  int t = blockIdx.x;
  const int co_t = t % p.co_tiles;
  const int u0 = (t / p.co_tiles) * MT;
  const int nu = min(MT, p.ntaps * p.ci_tiles - u0);
  const int tap = u0 / p.ci_tiles;               // unit 0's tap: selects the dY view (equal for all units, host-checked)
  const int split = blockIdx.y;
  const int kb0 = split * p.kb_per_split;
  const int kb1 = min(p.kblocks, kb0 + p.kb_per_split);
  const int num_kb = kb1 - kb0;                 // >= 1 by construction
  const int co0 = co_t * BN;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], WG_CWARPS);      // one arrive per consumer warp
    }
    for (int b = 0; b < 2; ++b) mbar_init(&buf_free[b], WG_CWARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (PART) {
    // a box of fewer than 32 pixels fills the same leading rows of every 4 KB box slot of the ring: zero the others once,
    // so the A fragments and the transposed dY tile hold zeros for the k-block's missing pixels
    const int tail = (WG_P - p.rows_used) * 128;
    const int words = p.stages * (stage_bytes / WG_BOX) * (tail / 16);
    for (int i = threadIdx.x; i < words; i += WG_THREADS) {
      const int slot = i / (tail / 16), off = i % (tail / 16);
      sts128(smem_u32(smem + slot * WG_BOX + p.rows_used * 128) + off * 16, make_float4(0.f, 0.f, 0.f, 0.f));
    }
  }
  __syncthreads();

  // a 256-column accumulator (128 registers a thread) plus its A fragments needs more than the 168 registers a thread
  // that 384 threads leave: the producer warpgroup hands most of its registers to the consumers
  constexpr bool REALLOC = MT * BN >= 256;
  if (warp >= WG_CWARPS) {
    if (REALLOC) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == WG_CWARPS && lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_x.m[p.amap[tap]]) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tm_dy.m[p.bmap[tap]]) : "memory");
      const CUtensorMap* mb = &tm_dy.m[p.bmap[tap]];
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        int r = kb;
        const int tw = r % p.tiles_w; r /= p.tiles_w;
        const int th = r % p.tiles_h;
        const int tn = r / p.tiles_h;
        const int w0 = tw * p.bw, h0 = th * p.bh, n0 = tn * p.bni;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * stage_bytes;
        uint8_t* sb = sa + a_bytes;
        mbar_expect_tx(&full_bar[stage], PART ? (uint32_t)((nu * 4 + BN / 32) * p.rows_used * 128)
                                              : (uint32_t)(nu * WG_A_BYTES + b_bytes));
        for (int i = 0; i < nu; ++i) {
          const int u = u0 + i, utap = u / p.ci_tiles, ci0 = (u % p.ci_tiles) * 128;
          const CUtensorMap* ma = &tm_x.m[p.amap[utap]];
#pragma unroll
          for (int g = 0; g < 4; ++g)
            tma_load_4d(sa + i * WG_A_BYTES + g * WG_BOX, ma, &full_bar[stage], ci0 + g * 32, w0 + p.off_w[utap],
                        h0 + p.off_h[utap], n0);
        }
        for (int g = 0; g < BN / 32; ++g) tma_load_4d(sb + g * WG_BOX, mb, &full_bar[stage], co0 + g * 32, w0, h0, n0);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===== consumer warpgroups =====
  if (REALLOC) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  // The MT x 4 MMAs of a k-block (unit i / 4, k-step i % 4) go out in two commit groups of GK, each fed by its own A
  // fragment registers.  k-block kb:
  //   wait for G0 of kb - 1 (G1 of kb - 1 still runs) | load G0's fragments of kb | wait until dY buffer kb & 1 is free |
  //   transpose the stage's dY into it | CTA barrier (both halves of the dY tile written and visible to the async proxy) |
  //   issue G0 of kb | wait for G1 of kb - 1 (G0 of kb runs), which frees buffer (kb - 1) & 1 | load G1's fragments of
  //   kb | release the stage | issue G1 of kb.
  // Fragment registers are rewritten only once the MMAs that read them have retired; a dY buffer only once both
  // warpgroups' MMAs of two k-blocks back have (buf_free: one arrive per consumer warp).  Each accumulator receives its
  // MMAs in unit-major, k-step order, k-block after k-block.
  constexpr int GK = 2 * MT;
  const int wg = warp >> 2;
  const int cib = wg_a_channel(warp, lane), q = lane & 3;
  const uint32_t a_box = (2 * wg + ((warp >> 1) & 1)) * WG_BOX + (cib & 3) * 4;
  const uint32_t a_lo = a_box + q * 128 + ((((cib >> 2) ^ q) & 7) << 4);                // pixel 8k + q
  const uint32_t a_hi = a_box + (q + 4) * 128 + ((((cib >> 2) ^ (q + 4)) & 7) << 4);    // pixel 8k + q + 4
  const bool all_units = MT == 1 || nu == MT;   // uniform over the CTA: the last tile of an odd unit count has one
  float acc[MT][BN / 2];
#pragma unroll
  for (int u = 0; u < MT; ++u)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[u][i] = 0.f;
  uint32_t fa[2][GK][4];
  int stage = 0;
  uint32_t phase = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int h = kb & 1;
    mbar_wait(&full_bar[stage], phase);
    const uint32_t s_addr = smem_u32(smem + stage * stage_bytes);
    const uint32_t t_addr = smem_u32(tbuf + h * b_bytes);
    wgmma_wait<1>();                              // G0 of kb - 1 retired
    wg_load_a<GK>(fa[0], s_addr, a_lo, a_hi, p.round_a);
    if (kb >= 2) mbar_wait(&buf_free[h], ((kb >> 1) & 1) ^ 1);
    wg_transpose<BN>(t_addr, s_addr + a_bytes, p.round_b, warp, lane);
    fence_proxy_async();
    named_bar(1, 32 * WG_CWARPS);
#pragma unroll
    for (int u = 0; u < MT; ++u)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc_fence(acc[u][i]);
    wgmma_fence();
#pragma unroll
    for (int e = 0; e < GK; ++e)                  // 8 pixels (32 B of every dY row) per MMA
      wgmma_tf32_rs<BN>(acc[e / 4], fa[0][e], make_desc(t_addr + (e % 4) * 32));
    wgmma_commit();
    wgmma_wait<1>();                              // G1 of kb - 1 retired: its dY buffer is free
    if (kb >= 1 && lane == 0) mbar_arrive(&buf_free[h ^ 1]);
    if (all_units) wg_load_a<GK>(fa[1], s_addr + (GK / 4) * WG_A_BYTES + (GK % 4) * 1024, a_lo, a_hi, p.round_a);
    // the warp's reads of the TMA stage are complete (fragments loaded, dY values stored): release it to the producer
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    wgmma_fence();
    if (all_units) {                              // a CTA past the last unit issues no MMAs for it
#pragma unroll
      for (int e = 0; e < GK; ++e)
        wgmma_tf32_rs<BN>(acc[(GK + e) / 4], fa[1][e], make_desc(t_addr + ((GK + e) % 4) * 32));
    }
    wgmma_commit();
    if (++stage == p.stages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
#pragma unroll
  for (int u = 0; u < MT; ++u)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc_fence(acc[u][i]);
  // epilogue: accumulator rows lane / 4 and lane / 4 + 8 are channels ci = cib, cib + 1 of the thread's box (see
  // wg_a_channel), columns co0 + 8j + 2 (lane % 4) + {0, 1}
  const int c2 = (lane & 3) * 2;
  const bool vec2 = (p.cout & 1) == 0;
#pragma unroll
  for (int u = 0; u < MT; ++u) {
    if (u >= nu) continue;
    const int uu = u0 + u, utap = uu / p.ci_tiles, ci0 = (uu % p.ci_tiles) * 128;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = (2 * wg + ((warp >> 1) & 1)) * 32 + cib + h;
      if (ci0 + row >= p.cin) continue;          // the last ci tile may hang over Cin (TMA zero-filled those channels)
      float* orow = p.partial + (((long long)split * p.taps_total + p.wtap[utap]) * p.cin + ci0 + row) * p.cout + co0;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = j * 8 + c2;
        if (co0 + c >= p.cout) continue;         // Cout zero-padded to the 32-column tile (e.g. 24-wide projections)
        if (vec2) {
          *reinterpret_cast<float2*>(orow + c) = make_float2(acc[u][4 * j + 2 * h], acc[u][4 * j + 2 * h + 1]);
        } else {
          orow[c] = acc[u][4 * j + 2 * h];
          if (co0 + c + 1 < p.cout) orow[c + 1] = acc[u][4 * j + 2 * h + 1];
        }
      }
    }
  }
}

// the n x h x w pixel grid cut into 32-pixel TMA boxes of bw x bh x bni
bool box32(int n, int h, int w, int* bw, int* bh, int* bni) {
  if (n < 1 || h < 1 || w < 1) return false;
  int b = w < 32 ? w : 32;
  if (32 % b != 0 || w % b != 0) return false;
  int hh = 32 / b; if (hh > h) hh = h;
  if (h % hh != 0) return false;
  int ni = 32 / (b * hh);
  if (ni < 1 || b * hh * ni != 32 || n % ni != 0) return false;
  *bw = b; *bh = hh; *bni = ni;
  return true;
}

// A grid whose width neither divides 32 nor is a multiple of it: the box of at most 32 pixels, no larger than the grid in
// any dimension, that needs the fewest k-blocks (ties: the wider box).  At batch 64: 48 -> 16x2, 24 -> 8x4, 12 -> 4x4 x 2
// images, 6 -> 2x2 x 8, 3 -> 1x1 x 32, every MMA row a real pixel; at batch 4, 3 -> 3x3 x 3 (27 rows, the second image
// tile half past the batch).  Every other width keeps box32's answer, or its refusal.
bool box_any(int n, int h, int w, int* bw, int* bh, int* bni) {
  if (n < 1 || h < 1 || w < 1 || 32 % w == 0 || w % 32 == 0) return false;
  long long best = -1;
  for (int b = w < 32 ? w : 32; b >= 1; --b)
    for (int hh = 32 / b < h ? 32 / b : h; hh >= 1; --hh) {
      const int ni = 32 / (b * hh) < n ? 32 / (b * hh) : n;
      const long long kb = (long long)((w + b - 1) / b) * ((h + hh - 1) / hh) * ((n + ni - 1) / ni);
      if (best < 0 || kb < best) { best = kb; *bw = b; *bh = hh; *bni = ni; }
    }
  return true;
}

// the box the kernel takes for an n x h x w grid; per-image launches (one k-block range per image) take box32's only
bool wg_box(int n, int h, int w, bool per_image, int* bw, int* bh, int* bni) {
  return box32(n, h, w, bw, bh, bni) || (!per_image && box_any(n, h, w, bw, bh, bni));
}

int pick_bn(int ncols) {
  if (ncols <= 256 && ncols % 4 == 0) return (ncols + 31) / 32 * 32;     // zero-padded tile, stores are masked
  if (ncols % 32) return 0;
  if (ncols <= 256) return ncols;
  if (ncols % 256 == 0) return 256;
  if (ncols % 192 == 0) return 192;
  if (ncols % 128 == 0) return 128;
  return 0;
}

// TMA ring depth for a shared-memory budget (ring + the two transposed dY tiles; the barrier placement in the consumer
// loop lets the transpose overlap the MMAs without a third one); returns the dynamic smem size.  At one CTA per SM a
// 48 KB stage (BN 256 with MT 1, or BN 128 with MT 2) gets a 3- or 4-deep ring.
size_t wg_smem(size_t stage_bytes, size_t t_bytes, size_t budget, int* stages) {
  long long s = ((long long)budget - 2 * (long long)t_bytes) / (long long)stage_bytes;
  if (s > WG_MAX_STAGES) s = WG_MAX_STAGES;
  if (s < 2) s = 2;
  *stages = (int)s;
  return (size_t)s * stage_bytes + 2 * t_bytes + 1024 + 256;
}

template <int BN, int MT, bool PART>
int wg_launch_t(cgan_ctx* ctx, dim3 grid, size_t smem, const BMaps& tm_x, const BMaps& tm_dy, const WgParams& p) {
  static bool attr_set = false;
  if (!attr_set) {
    CGAN_CUDA(ctx, cudaFuncSetAttribute(wgrad_tc_kernel<BN, MT, PART>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        227 * 1024));
    attr_set = true;
  }
  wgrad_tc_kernel<BN, MT, PART><<<grid, WG_THREADS, smem, ctx->stream>>>(tm_x, tm_dy, p);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

// one instantiation per (bn, mt, partial box): the accumulator fragment is sized at compile time
int wg_launch(cgan_ctx* ctx, dim3 grid, size_t smem, const BMaps& tm_x, const BMaps& tm_dy, const WgParams& p) {
#define WG_CASE(BN, MT)                                                                                        \
  if (p.bn == BN && p.mt == MT)                                                                                \
    return p.rows_used < WG_P ? wg_launch_t<BN, MT, true>(ctx, grid, smem, tm_x, tm_dy, p)                    \
                              : wg_launch_t<BN, MT, false>(ctx, grid, smem, tm_x, tm_dy, p);
  WG_CASE(32, 1) WG_CASE(64, 1) WG_CASE(96, 1) WG_CASE(128, 1) WG_CASE(160, 1) WG_CASE(192, 1) WG_CASE(224, 1)
  WG_CASE(256, 1) WG_CASE(32, 2) WG_CASE(64, 2) WG_CASE(96, 2) WG_CASE(128, 2)
#undef WG_CASE
  return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: no kernel for this column tile%s", "cgan_wgrad_tc");
}

}  // namespace

bool cgan_wgrad_tc_fits(const TcWgrad& g) {
  int bw, bh, bni;
  return wg_box(g.dy.n, g.dy.h, g.dy.w, g.per_image, &bw, &bh, &bni) && (!g.per_image || (bni == 1 && g.dy.n <= 65535)) &&
         g.x.ch > 0 && g.x.ch % 32 == 0 &&            // ci tiles of 128, the last one zero-padded
         pick_bn(g.dy.ch) != 0 && g.taps.ntaps >= 1 && g.taps.ntaps <= WG_MAX_TAPS && al16(g.x.in) && al16(g.dy.in) &&
         al16(g.dw);
}

int cgan_wgrad_tc(cgan_ctx* ctx, const TcWgrad& g) {
  if (!cgan_wgrad_tc_fits(g)) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: shape%s", "cgan_wgrad_tc");
  WgParams p;
  memset(&p, 0, sizeof(p));
  const int n = g.dy.n, gh = g.dy.h, gw = g.dy.w;      // the pixel grid
  p.round_a = g.x.tf32 ? 0 : 1;
  p.round_b = g.dy.tf32 ? 0 : 1;
  wg_box(n, gh, gw, g.per_image, &p.bw, &p.bh, &p.bni);
  p.rows_used = p.bw * p.bh * p.bni;
  p.tiles_w = (gw + p.bw - 1) / p.bw;
  p.tiles_h = (gh + p.bh - 1) / p.bh;
  p.kblocks = (int)((long long)p.tiles_w * p.tiles_h * ((n + p.bni - 1) / p.bni));    // n * gh * gw / 32 for box32
  p.bn = pick_bn(g.dy.ch);
  p.ci_tiles = (g.x.ch + 127) / 128;
  p.co_tiles = (g.dy.ch + p.bn - 1) / p.bn;
  p.cin = g.x.ch; p.cout = g.dy.ch; p.taps_total = g.taps_total;
  // tap i pairs x view amap[i] at [y + off_h, x + off_w] with dy view bmap[i] at [y, x]
  const ConvTaps& t = g.taps;
  p.ntaps = t.ntaps;
  for (int i = 0; i < t.ntaps; ++i) {
    p.off_h[i] = t.off_h[i]; p.off_w[i] = t.off_w[i]; p.wtap[i] = t.wtap[i];
    p.amap[i] = g.taps_view_dy ? 0 : t.view[i];
    p.bmap[i] = g.taps_view_dy ? t.view[i] : 0;
  }
  // two (tap, ci-tile) units per CTA when they read the same dY view: dY is then fetched once per k-block for both
  const int units = p.ci_tiles * t.ntaps;
  bool same_b = true;
  for (int i = 1; i < t.ntaps; ++i) same_b = same_b && p.bmap[i] == p.bmap[0];
  p.mt = (!g.per_image && ctx->tc_mt_max >= 2 && same_b && units >= 2 && 2 * p.bn <= WG_ACC_COLS) ? 2 : 1;
  const size_t t_bytes = (size_t)(p.bn / 32) * WG_BOX;
  const size_t stage_bytes = (size_t)p.mt * WG_A_BYTES + t_bytes;
  const long long tiles = (long long)p.co_tiles * ((units + p.mt - 1) / p.mt);
  int splits;
  size_t smem;
  if (g.per_image) {
    // "split" i = image i: its partial tile IS the result dw[i]
    p.kb_per_split = gh * gw / WG_P;
    splits = n;
    smem = wg_smem(stage_bytes, t_bytes, 110 * 1024, &p.stages);
  } else {
    // stages of up to 24 KB (BN <= 64 with MT 1) run two CTAs per SM
    const bool two_ctas = stage_bytes <= 24 * 1024;
    // two CTAs per SM in total (two waves when only one fits), rounded DOWN so the grid never spills a few CTAs into an
    // extra wave; the pixel chain each fp32 accumulator sums stays as short as with two resident CTAs per SM
    splits = (int)((2ll * ctx->num_sms) / tiles);
    int max_splits = p.kblocks / 8 > 0 ? p.kblocks / 8 : 1;
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    p.kb_per_split = (p.kblocks + splits - 1) / splits;
    splits = (p.kblocks + p.kb_per_split - 1) / p.kb_per_split;
    smem = wg_smem(stage_bytes, t_bytes, two_ctas ? 110 * 1024 : 225 * 1024, &p.stages);
  }

  const bool reduce = !g.per_image && splits > 1;
  const long long wn = (long long)p.taps_total * p.cin * p.cout;
  p.partial = g.dw;
  if (reduce) {
    void* ws = nullptr;
    int rc = cgan_ws(ctx, (size_t)splits * wn * sizeof(float), &ws);
    if (rc) return rc;
    p.partial = reinterpret_cast<float*>(ws);
  }

  BMaps tm_x, tm_dy;
  memset(&tm_x, 0, sizeof(tm_x));
  memset(&tm_dy, 0, sizeof(tm_dy));
  for (int v = 0; v < 4; ++v)
    if (!make_view_map(&tm_x.m[v], g.x, v, p.bw, p.bh, p.bni, CU_TENSOR_MAP_SWIZZLE_128B) ||
        !make_view_map(&tm_dy.m[v], g.dy, v, p.bw, p.bh, p.bni, CU_TENSOR_MAP_SWIZZLE_NONE))
      return cgan_fail(ctx, CGAN_ERR_CUDA, "%s: cuTensorMapEncodeTiled failed%s", "cgan_wgrad_tc");
  int rc = wg_launch(ctx, dim3((unsigned)tiles, (unsigned)splits), smem, tm_x, tm_dy, p);
  if (rc || !reduce) return rc;
  return cgan_splitk_reduce(ctx, g.dw, p.partial, wn, splits);
}
