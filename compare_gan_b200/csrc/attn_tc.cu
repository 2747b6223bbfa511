// Fused self-attention of the non-local block (arch_ops.py:734-753) on warpgroup MMAs (wgmma, sm_90a) — math_mode 1.
//
//   O[i] = softmax(Q[i] K[i]^T) V[i]          Q = theta [Lq, dk], K = phi [Lk, dk], V = g [Lk, dv] per image i
//
// The reference materialises the [Lq, Lk] score matrix (tf.matmul -> tf.nn.softmax -> tf.matmul); at BigGAN-128 that is
// 4096 x 1024 floats per image, 4.3 GB per batch of 256, crossing HBM three times per direction.  Here the scores never
// leave the registers: a score tile is a wgmma accumulator fragment, exponentiated and rounded to TF32 in place, and the
// second MMA takes it as its A operand straight from the registers.
//
// A CTA is two consumer warpgroups (256 threads), warpgroup g owning rows 64g..64g+63 of a 128-row tile; operand tiles are
// staged in shared memory as 128B-swizzled K-major tiles (wgmma takes 32-bit operands only K-major) by all 256 threads.
// Forward (attn_fwd_kernel): one CTA per 128 queries of one image, key tiles of 64.
//   pass 1: S_j = Q K_j^T (m64n64k8, dk zero-padded to 32) -> row maxima m.
//   pass 2: S_j again (K has 4x fewer channels than V: recomputing costs 1/4 of the P V MMAs and avoids rescaling O),
//           p = exp(s - m), l += p, O += P V_j.  Epilogue: O / l, lse = m + log l (kept for the backward).
// Backward: P is recomputed from Q, K and lse (no [Lq, Lk] tensor is ever stored); with D = rowsum(dO * O),
//   dS = P * (dP - D),  dP = dO V^T,  dQ = dS K,  dK = dS^T Q,  dV = P^T dO.
//   attn_bwd_dq_kernel: one CTA per 128 queries, loops over key tiles (accumulates dQ in registers);
//   attn_bwd_dkv_kernel: one CTA per 128 keys, loops over query tiles of 64 (accumulates dK, dV) — S^T and dP^T are produced
//   directly (M = keys), so no transposition of a score tile exists and the summation order is fixed (deterministic).
//
// A register operand P (or dS) of key columns 8s..8s+7 is the accumulator fragment itself: this thread holds columns
// 8s + 2t and 8s + 2t + 1 (t = lane % 4), which the A fragment places at k = t and k = t + 4.  The B operand of such an MMA
// (V, K, dO or Q, transposed into [channel][row] tiles) therefore stores row 8s + r at k position r / 2 + 4 (r & 1).
//
// Operands are consumed as TF32: callers pass tensors already rounded to the nearest TF32 value (cgan_round_tf32 or a
// producer's ROUND_OUT epilogue).  Accumulation is fp32.  Where the kernels round, per score (i, j) of image b:
//   s  = Q_i . K_j (fp32 accumulation)     p = ex2.approx.ftz(s log2e - m_i log2e), m_i the row maximum (forward) or
//                                              ex2.approx.ftz(s log2e - lse_i log2e) (both backward kernels)
//   forward:  l_i = sum_j p (fp32, p UNROUNDED),  O_i = (sum_j rna_tf32(p) V_j) / l_i,  lse_i = m_i + log l_i
//   backward: dS = rna_tf32(p (dP - D_i)) from the UNROUNDED p in both kernels, dQ = dS K, dK = dS^T Q,
//             dV = rna_tf32(p)^T dO
// so the normaliser is the one lse describes, and dQ and dK are contractions of the same dS.  tests/abi_emulator.py
// (attention_tf32_model) is this contract in numpy.
//
// Memory: q, k, v and dout are read as float4 (16-byte aligned), out, dq, dk and dv stored and lse read as float2 (8-byte
// aligned); the entry points refuse other pointers with CGAN_ERR_UNSUPPORTED before launching anything.
#include "tc_common.cuh"

namespace {

using namespace tc;

constexpr int AT_THREADS = 256;     // two consumer warpgroups
constexpr int AT_TQ = 128;          // rows per CTA
constexpr int AT_TK = 64;           // columns per score tile (wgmma N of the score MMAs)
constexpr int AT_DK = 32;           // dk zero-padded to one 128-byte swizzle row
constexpr float AT_LOG2E = 1.4426950408889634f;
constexpr size_t AT_SMEM_MAX = 227 * 1024;

struct AtParams {
  int lq, lk, dk, dv;
  float* out;           // fwd: O          dq: dQ        dkv: dK
  float* out2;          // fwd: lse        dq: -         dkv: dV
  const float* lse;     // bwd
  const float* dsum;    // bwd: D = rowsum(dO * O)
};

// round to the nearest TF32 value, ties away from zero — bit-identical to cvt.rna.tf32.f32 for finite values below the
// largest TF32 binade (probabilities and their products here), in two integer ops
__device__ __forceinline__ float rnd_tf32(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void at_sync() { named_bar(1, AT_THREADS); }

// [rows][ch] fp32 rows (ld = ch) -> K-major tile of `rows` x kpad (kpad / 32 chunks of rows x 128 B), zero beyond ch
__device__ __forceinline__ void load_k(uint32_t dst, int rows, int kpad, const float* src, int ch) {
  const int q4 = kpad / 4;
  for (int e = threadIdx.x; e < rows * q4; e += AT_THREADS) {
    const int r = e / q4, c = (e - r * q4) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < ch) v = __ldg(reinterpret_cast<const float4*>(src + (size_t)r * ch + c));
    sts128(dst + (c >> 5) * rows * 128 + sw128_offset(r, c & 31), v);
  }
}

// [AT_TK rows][ch] -> transposed K-major tile [npad channels][AT_TK rows]: the B operand of an MMA whose A operand is a
// register score fragment (row 8s + r of the source at k position 8s + r / 2 + 4 (r & 1), see the header)
__device__ __forceinline__ void load_t(uint32_t dst, int npad, const float* src, int ch) {
  const int q4 = npad / 4;
  for (int e = threadIdx.x; e < AT_TK * q4; e += AT_THREADS) {
    const int r = e / q4, c = (e - r * q4) * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < ch) v = __ldg(reinterpret_cast<const float4*>(src + (size_t)r * ch + c));
    const int pos = (r & ~7) + ((r & 7) >> 1) + ((r & 1) << 2);
    const uint32_t base = dst + (pos >> 5) * npad * 128;
    const int k = pos & 31;
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(base + sw128_offset(c, k)), "f"(v.x) : "memory");
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(base + sw128_offset(c + 1, k)), "f"(v.y) : "memory");
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(base + sw128_offset(c + 2, k)), "f"(v.z) : "memory");
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(base + sw128_offset(c + 3, k)), "f"(v.w) : "memory");
  }
}

template <int N>
__device__ __forceinline__ void zero(float (&a)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) a[i] = 0.f;
}
template <int N>
__device__ __forceinline__ void fence_acc(float (&a)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) acc_fence(a[i]);
}

// acc (m64 x N, this warpgroup's rows) += A (tile of `arows` rows, this warpgroup's 64 of them, K = 8 * KSTEPS) * B^T
// (tile of N rows); both K-major in chunks of 32
template <int N, int KSTEPS>
__device__ __forceinline__ void mma_ss(float* acc, uint32_t a, int arows, int wg, uint32_t b) {
#pragma unroll
  for (int s = 0; s < KSTEPS; ++s)
    wgmma_tf32<N>(acc, make_desc(a + (s >> 2) * arows * 128 + wg * 64 * 128 + (s & 3) * 32),
                  make_desc(b + (s >> 2) * N * 128 + (s & 3) * 32));
}
// acc (m64 x N) += P (register fragment of a 64-column score tile) * B, B = transposed tile [N][AT_TK] from load_t
template <int N>
__device__ __forceinline__ void mma_rs(float* acc, const float (&p)[32], uint32_t b) {
#pragma unroll
  for (int s = 0; s < AT_TK / 8; ++s) {
    const uint32_t a[4] = {__float_as_uint(p[4 * s]), __float_as_uint(p[4 * s + 2]), __float_as_uint(p[4 * s + 1]),
                           __float_as_uint(p[4 * s + 3])};
    wgmma_tf32_rs<N>(acc, a, make_desc(b + (s >> 2) * N * 128 + (s & 3) * 32));
  }
}

// store rows (r, r + 8) x columns 8j + 2t + {0,1} < ncols of an m64 x N fragment into out[row][ld]
template <int N>
__device__ __forceinline__ void store_frag(float* out, int ld, int ncols, int row, const float* acc, float s0, float s1) {
  const int c2 = (threadIdx.x & 3) * 2;
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    const int c = 8 * j + c2;
    if (c < ncols) {        // ncols is a multiple of 4: both columns exist
      *reinterpret_cast<float2*>(out + (size_t)row * ld + c) = make_float2(acc[4 * j] * s0, acc[4 * j + 1] * s0);
      *reinterpret_cast<float2*>(out + (size_t)(row + 8) * ld + c) = make_float2(acc[4 * j + 2] * s1, acc[4 * j + 3] * s1);
    }
  }
}

template <int NV>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_fwd_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v, const AtParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sq = smem_u32(smem);                  // [128][32]
  const uint32_t sk = sq + AT_TQ * 128;                // [64][32]
  const uint32_t svt = sk + AT_TK * 128;               // [NV][64] transposed, permuted
  const int img = blockIdx.y, q0 = blockIdx.x * AT_TQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const float* kimg = k + (size_t)img * p.lk * p.dk;
  const float* vimg = v + (size_t)img * p.lk * p.dv;
  const int ntiles = p.lk / AT_TK;

  load_k(sq, AT_TQ, AT_DK, q + ((size_t)img * p.lq + q0) * p.dk, p.dk);
  float s[32];
  float m0 = -INFINITY, m1 = -INFINITY;
  for (int j = 0; j < ntiles; ++j) {                   // pass 1: row maxima
    load_k(sk, AT_TK, AT_DK, kimg + (size_t)j * AT_TK * p.dk, p.dk);
    fence_proxy_async();
    at_sync();
    zero(s);
    fence_acc(s);
    wgmma_fence();
    mma_ss<AT_TK, AT_DK / 8>(s, sq, AT_TQ, wg, sk);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(s);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      m0 = fmaxf(m0, fmaxf(s[4 * i], s[4 * i + 1]));
      m1 = fmaxf(m1, fmaxf(s[4 * i + 2], s[4 * i + 3]));
    }
    at_sync();
  }
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
  const float mb0 = m0 * AT_LOG2E, mb1 = m1 * AT_LOG2E;
  float o[NV / 2];
  zero(o);
  float l0 = 0.f, l1 = 0.f;
  for (int j = 0; j < ntiles; ++j) {                   // pass 2: probabilities and O
    load_k(sk, AT_TK, AT_DK, kimg + (size_t)j * AT_TK * p.dk, p.dk);
    load_t(svt, NV, vimg + (size_t)j * AT_TK * p.dv, p.dv);
    fence_proxy_async();
    at_sync();
    zero(s);
    fence_acc(s);
    wgmma_fence();
    mma_ss<AT_TK, AT_DK / 8>(s, sq, AT_TQ, wg, sk);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(s);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float p0 = ex2(fmaf(s[4 * i], AT_LOG2E, -mb0)), p1 = ex2(fmaf(s[4 * i + 1], AT_LOG2E, -mb0));
      const float p2 = ex2(fmaf(s[4 * i + 2], AT_LOG2E, -mb1)), p3 = ex2(fmaf(s[4 * i + 3], AT_LOG2E, -mb1));
      l0 += p0 + p1; l1 += p2 + p3;
      s[4 * i] = rnd_tf32(p0); s[4 * i + 1] = rnd_tf32(p1); s[4 * i + 2] = rnd_tf32(p2); s[4 * i + 3] = rnd_tf32(p3);
    }
    fence_acc(o);
    wgmma_fence();
    mma_rs<NV>(o, s, svt);
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(o);
    at_sync();
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const size_t r0 = (size_t)img * p.lq + q0 + row;
  store_frag<NV>(p.out + r0 * p.dv, p.dv, p.dv, 0, o, 1.f / l0, 1.f / l1);
  if ((lane & 3) == 0) {
    p.out2[r0] = m0 + logf(l0);
    p.out2[r0 + 8] = m1 + logf(l1);
  }
}

template <int NV>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_bwd_dq_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                   const float* __restrict__ dout, const AtParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sq = smem_u32(smem);                  // [128][32]
  const uint32_t sdo = sq + AT_TQ * 128;               // [128][NV]
  const uint32_t sk = sdo + AT_TQ * NV * 4;            // [64][32]
  const uint32_t sv = sk + AT_TK * 128;                // [64][NV]
  const uint32_t skt = sv + AT_TK * NV * 4;            // [32][64] transposed, permuted
  const int img = blockIdx.y, q0 = blockIdx.x * AT_TQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const size_t r0 = (size_t)img * p.lq + q0 + row;
  const float* kimg = k + (size_t)img * p.lk * p.dk;
  const float* vimg = v + (size_t)img * p.lk * p.dv;
  const float lb0 = p.lse[r0] * AT_LOG2E, lb1 = p.lse[r0 + 8] * AT_LOG2E;
  const float d0 = p.dsum[r0], d1 = p.dsum[r0 + 8];

  load_k(sq, AT_TQ, AT_DK, q + ((size_t)img * p.lq + q0) * p.dk, p.dk);
  load_k(sdo, AT_TQ, NV, dout + ((size_t)img * p.lq + q0) * p.dv, p.dv);
  float s[32], dp[32], dq[AT_DK / 2];
  zero(dq);
  for (int j = 0; j < p.lk / AT_TK; ++j) {
    load_k(sk, AT_TK, AT_DK, kimg + (size_t)j * AT_TK * p.dk, p.dk);
    load_k(sv, AT_TK, NV, vimg + (size_t)j * AT_TK * p.dv, p.dv);
    load_t(skt, AT_DK, kimg + (size_t)j * AT_TK * p.dk, p.dk);
    fence_proxy_async();
    at_sync();
    zero(s); zero(dp);
    fence_acc(s); fence_acc(dp);
    wgmma_fence();
    mma_ss<AT_TK, AT_DK / 8>(s, sq, AT_TQ, wg, sk);       // S = Q K^T
    mma_ss<AT_TK, NV / 8>(dp, sdo, AT_TQ, wg, sv);        // dP = dO V^T
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(s); fence_acc(dp);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const bool lo = (i & 2) == 0;
      const float pr = ex2(fmaf(s[i], AT_LOG2E, -(lo ? lb0 : lb1)));
      s[i] = rnd_tf32(pr * (dp[i] - (lo ? d0 : d1)));      // dS
    }
    fence_acc(dq);
    wgmma_fence();
    mma_rs<AT_DK>(dq, s, skt);                            // dQ += dS K
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(dq);
    at_sync();
  }
  store_frag<AT_DK>(p.out + r0 * p.dk, p.dk, p.dk, 0, dq, 1.f, 1.f);
}

template <int NV>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_bwd_dkv_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                    const float* __restrict__ dout, const AtParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t sk = smem_u32(smem);                  // [128 keys][32]
  const uint32_t sv = sk + AT_TQ * 128;                // [128 keys][NV]
  const uint32_t sq = sv + AT_TQ * NV * 4;             // [64 queries][32]
  const uint32_t sdo = sq + AT_TK * 128;               // [64 queries][NV]
  const uint32_t sdot = sdo + AT_TK * NV * 4;          // [NV][64] transposed, permuted
  const uint32_t sqt = sdot + AT_TK * NV * 4;          // [32][64] transposed, permuted
  const int img = blockIdx.y, k0 = blockIdx.x * AT_TQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c2 = (lane & 3) * 2;
  const float* qimg = q + (size_t)img * p.lq * p.dk;
  const float* doimg = dout + (size_t)img * p.lq * p.dv;

  load_k(sk, AT_TQ, AT_DK, k + ((size_t)img * p.lk + k0) * p.dk, p.dk);
  load_k(sv, AT_TQ, NV, v + ((size_t)img * p.lk + k0) * p.dv, p.dv);
  float s[32], dp[32], dk[AT_DK / 2], dv[NV / 2];
  zero(dk); zero(dv);
  for (int j = 0; j < p.lq / AT_TK; ++j) {
    const float* qj = qimg + (size_t)j * AT_TK * p.dk;
    const float* doj = doimg + (size_t)j * AT_TK * p.dv;
    load_k(sq, AT_TK, AT_DK, qj, p.dk);
    load_k(sdo, AT_TK, NV, doj, p.dv);
    load_t(sdot, NV, doj, p.dv);
    load_t(sqt, AT_DK, qj, p.dk);
    fence_proxy_async();
    at_sync();
    zero(s); zero(dp);
    fence_acc(s); fence_acc(dp);
    wgmma_fence();
    mma_ss<AT_TK, AT_DK / 8>(s, sk, AT_TQ, wg, sq);       // S^T = K Q^T
    mma_ss<AT_TK, NV / 8>(dp, sv, AT_TQ, wg, sdo);        // dP^T = V dO^T
    wgmma_commit();
    // lse / D of this thread's query columns while the MMAs run
    const size_t qr = (size_t)img * p.lq + (size_t)j * AT_TK;
    float lb[16], dd[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float2 l2 = *reinterpret_cast<const float2*>(p.lse + qr + 8 * i + c2);
      const float2 d2 = *reinterpret_cast<const float2*>(p.dsum + qr + 8 * i + c2);
      lb[2 * i] = l2.x * AT_LOG2E; lb[2 * i + 1] = l2.y * AT_LOG2E;
      dd[2 * i] = d2.x; dd[2 * i + 1] = d2.y;
    }
    wgmma_wait<0>();
    fence_acc(s); fence_acc(dp);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = 2 * (i >> 2) + (i & 1);
      const float pr = ex2(fmaf(s[i], AT_LOG2E, -lb[col]));
      dp[i] = rnd_tf32(pr * (dp[i] - dd[col]));            // dS^T, from the unrounded P as in attn_bwd_dq_kernel
      s[i] = rnd_tf32(pr);                                 // P^T
    }
    fence_acc(dv); fence_acc(dk);
    wgmma_fence();
    mma_rs<NV>(dv, s, sdot);                               // dV += P^T dO
    mma_rs<AT_DK>(dk, dp, sqt);                            // dK += dS^T Q
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(dv); fence_acc(dk);
    at_sync();
  }
  const size_t r0 = (size_t)img * p.lk + k0 + row;
  store_frag<AT_DK>(p.out + r0 * p.dk, p.dk, p.dk, 0, dk, 1.f, 1.f);
  store_frag<NV>(p.out2 + r0 * p.dv, p.dv, p.dv, 0, dv, 1.f, 1.f);
}

__global__ void round_tf32_kernel(float* __restrict__ y, const float* __restrict__ x, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = rna_tf32(x[i]);
}

bool shape_ok(int batch, int lq, int lk, int dk, int dv) {
  return batch >= 1 && batch <= 65535 && lq >= 128 && lq % 128 == 0 && lk >= 128 && lk % 128 == 0 && dk >= 4 && dk <= 32 &&
         dk % 4 == 0 && dv >= 16 && dv <= 128 && dv % 16 == 0;
}

void fill_params(AtParams* p, int lq, int lk, int dk, int dv) {
  memset(p, 0, sizeof(*p));
  p->lq = lq; p->lk = lk; p->dk = dk; p->dv = dv;
}

inline int nv_pad(int dv) { return (dv + 31) / 32 * 32; }      // V / dO columns zero-padded to whole swizzle rows

inline bool aligned(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

size_t fwd_smem(int nv) { return 1024 + AT_TQ * 128 + AT_TK * 128 + (size_t)AT_TK * nv * 4; }
size_t dq_smem(int nv) { return 1024 + AT_TQ * 128 + (size_t)AT_TQ * nv * 4 + AT_TK * 128 + (size_t)AT_TK * nv * 4 + AT_TK * 128; }
size_t dkv_smem(int nv) { return 1024 + AT_TQ * 128 + (size_t)AT_TQ * nv * 4 + AT_TK * 128 + 2 * (size_t)AT_TK * nv * 4 + AT_TK * 128; }

template <typename F>
int set_smem(cgan_ctx* ctx, F* kernel, size_t bytes, const char* who) {
  if (bytes > 227 * 1024) return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: shared memory%s", who);
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) return cgan_fail(ctx, CGAN_ERR_CUDA, "%s: %s", who, cudaGetErrorString(e));
  return CGAN_OK;
}

}  // namespace

extern "C" {

int cgan_round_tf32(cgan_ctx* ctx, float* y, const float* x, int64_t n) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, y && x && n >= 0, "bad argument");
  if (n == 0) return CGAN_OK;
  long long blocks = (n + 255) / 256, cap = (long long)ctx->num_sms * 16;
  round_tf32_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, ctx->stream>>>(y, x, n);
  CGAN_LAUNCHED(ctx);
  return CGAN_OK;
}

int cgan_attention_supported(cgan_ctx* ctx, int batch, int lq, int lk, int dk, int dv) {
  return (ctx && ctx->math_mode == 1 && shape_ok(batch, lq, lk, dk, dv)) ? 1 : 0;
}

int cgan_attention_fwd(cgan_ctx* ctx, const float* q, const float* k, const float* v, float* out, float* lse, int batch, int lq,
                       int lk, int dk, int dv) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, q && k && v && out && lse, "null pointer");
  if (!cgan_attention_supported(ctx, batch, lq, lk, dk, dv))
    return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: needs math_mode 1, lq, lk multiples of 128, dk <= 32 (x4), dv <= 128 (x16)%s",
                     "cgan_attention_fwd");
  if (!aligned(q, 16) || !aligned(k, 16) || !aligned(v, 16) || !aligned(out, 8) || !aligned(lse, 8))
    return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: needs q, k, v 16-byte aligned and out, lse 8-byte aligned%s",
                     "cgan_attention_fwd");
  AtParams p;
  fill_params(&p, lq, lk, dk, dv);
  p.out = out; p.out2 = lse;
  const int nv = nv_pad(dv);
  const size_t smem = fwd_smem(nv);
  const dim3 grid(lq / AT_TQ, batch);
  int rc;
#define AT_FWD(NV)                                                                    \
  case NV:                                                                            \
    rc = set_smem(ctx, attn_fwd_kernel<NV>, smem, "cgan_attention_fwd");              \
    if (rc) return rc;                                                                \
    attn_fwd_kernel<NV><<<grid, AT_THREADS, smem, ctx->stream>>>(q, k, v, p);         \
    break;
  switch (nv) { AT_FWD(32) AT_FWD(64) AT_FWD(96) AT_FWD(128) default: return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: dv%s", "cgan_attention_fwd"); }
#undef AT_FWD
  CGAN_LAUNCHED(ctx);
  ctx->last_path = CGAN_PATH_TCGEN05_TF32;
  return CGAN_OK;
}

int cgan_attention_bwd(cgan_ctx* ctx, const float* q, const float* k, const float* v, const float* out, const float* lse,
                       const float* dout, float* dq, float* dk_out, float* dv_out, int batch, int lq, int lk, int dk, int dv) {
  if (!ctx) return CGAN_ERR_ARG;
  CGAN_REQUIRE(ctx, q && k && v && out && lse && dout && dq && dk_out && dv_out, "null pointer");
  if (!cgan_attention_supported(ctx, batch, lq, lk, dk, dv))
    return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: unsupported shape or math mode%s", "cgan_attention_bwd");
  if (!aligned(q, 16) || !aligned(k, 16) || !aligned(v, 16) || !aligned(dout, 16) || !aligned(lse, 8) || !aligned(dq, 8) ||
      !aligned(dk_out, 8) || !aligned(dv_out, 8))
    return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED,
                     "%s: needs q, k, v, dout 16-byte aligned and lse, dq, dk, dv 8-byte aligned%s", "cgan_attention_bwd");
  void* ws = nullptr;
  int rc = cgan_ws(ctx, (size_t)batch * lq * sizeof(float), &ws);
  if (rc) return rc;
  float* dsum = reinterpret_cast<float*>(ws);
  rc = cgan_rowdot(ctx, dsum, dout, out, (int64_t)batch * lq, dv);          // D = rowsum(dO * O)
  if (rc) return rc;
  AtParams p;
  fill_params(&p, lq, lk, dk, dv);
  p.lse = lse; p.dsum = dsum;
  const int nv = nv_pad(dv);
  p.out = dq; p.out2 = nullptr;
  const dim3 gq(lq / AT_TQ, batch), gk(lk / AT_TQ, batch);
  const size_t sm_q = dq_smem(nv), sm_kv = dkv_smem(nv);
#define AT_BWD(NV)                                                                              \
  case NV:                                                                                      \
    rc = set_smem(ctx, attn_bwd_dq_kernel<NV>, sm_q, "cgan_attention_bwd");                     \
    if (rc) return rc;                                                                          \
    attn_bwd_dq_kernel<NV><<<gq, AT_THREADS, sm_q, ctx->stream>>>(q, k, v, dout, p);            \
    CGAN_LAUNCHED(ctx);                                                                         \
    p.out = dk_out; p.out2 = dv_out;                                                            \
    rc = set_smem(ctx, attn_bwd_dkv_kernel<NV>, sm_kv, "cgan_attention_bwd");                   \
    if (rc) return rc;                                                                          \
    attn_bwd_dkv_kernel<NV><<<gk, AT_THREADS, sm_kv, ctx->stream>>>(q, k, v, dout, p);          \
    CGAN_LAUNCHED(ctx);                                                                         \
    break;
  switch (nv) { AT_BWD(32) AT_BWD(64) AT_BWD(96) AT_BWD(128) default: return cgan_fail(ctx, CGAN_ERR_UNSUPPORTED, "%s: dv%s", "cgan_attention_bwd"); }
#undef AT_BWD
  ctx->last_path = CGAN_PATH_TCGEN05_TF32;
  return CGAN_OK;
}

}  // extern "C"
