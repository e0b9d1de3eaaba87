// Warpgroup-MMA (wgmma) / TMA GEMM for the codec's convs, transposed convs and linears.
//
//   D[(i,o), n] = sum_{tap} sum_{c} A[c, i + tap*tap_di, o*o_mul + tap*tap_do] * W[n, tap*Kc + c]
//
// A is a 3-D TMA tensor (c, i, o): the activation buffer itself (no im2col), so a causal conv is a
// K loop over taps.  A CTA computes 128 x BN output tiles, persistently: tiles blockIdx.x, +gridDim.x, ... with the N tile
// fastest, so CTAs running together share A rows in L2, and the TMA warp fetches the next tile's stages while the
// consumers run the epilogue of the current one.  Warp roles (288 threads): warpgroups 0 and 1 = consumers, each owning
// 64 rows of the tile; warp 8 = TMA producer filling an S-stage ring of [A fp32 128 x 32 | W_hi BN x 32 | W_lo BN x 32].
//
// Precision 0 ("3xTF32"): fp32-equivalent products for the encoder side, where RVQ indices must match the fp32 reference
// (SURVEY.md H1).  A consumer reads its A fragment out of the swizzled fp32 tile into registers, applies the fused
// pre-activation and splits each value x into hi = rna_tf32(x) and lo = rna_tf32(x - hi) (both exactly representable in
// TF32); the weights arrive pre-split.  Register-A wgmmas accumulate a_hi*b_hi into one accumulator and a_lo*b_hi +
// a_hi*b_lo into a second (the small terms kept apart; the 2^-22 lo*lo term is dropped).  Precision 1: one TF32 wgmma
// (hi only; the tensor core reads the top 19 bits of the fp32 weights).
// Every chunk of TC_CHUNK_STAGES stages (K = 128) starts fresh wgmma accumulators that are then added into fp32 registers
// with round-to-nearest, so the error of the tensor core's internal accumulation is bounded by one chunk, whatever K is.
//
// K-pair mode (a per-plan choice for launches with too few 128-row tiles to fill the SMs and a long K): a tile is 64 x BN
// and both consumer warpgroups hold the same 64 rows.  Warpgroup 0 computes the promotion chunks 0, 2, 4, ..., warpgroup
// 1 the chunks 1, 3, 5, ... and hands each chunk's d0 + d1, thread for thread, to warpgroup 0 through a two-slot
// shared-memory queue.  Warpgroup 0 adds the chunks into acc in chunk order, so every fp32 addition into acc is the one
// the 128-row mode makes and the output is bit-identical; it alone runs the epilogue.  The stage ring is split into one
// ring of S / 2 slots per warpgroup (a warpgroup that skipped the other's stages in one shared ring could wait on a
// slot two phases ahead), and the queue lives in the A halves the 64-row boxes leave unused.
#include <cstdlib>

#include "common.cuh"
#include "tc_common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {
extern void count_launch();
using namespace tc;

constexpr int TC_BM = 128;
constexpr int TC_BKE = 32;                 // fp32 elements per 128-byte swizzle row
constexpr int TC_A_BYTES = TC_BM * 128;    // 16 KB
constexpr int TC_CONSUMER_WARPS = 8;       // two warpgroups of 64 tile rows each
constexpr int TC_THREADS = 32 * TC_CONSUMER_WARPS + 32;   // + the TMA warp
constexpr int TC_CHUNK_STAGES = 4;         // K stages accumulated by the tensor core before promotion = 4 * 32

struct TcParams {
  float* C;
  float* C2;  // optional second output: act2(pre-activation value), same strides as C
  int act2;
  long long c_i_stride, c_o_stride, c_split_stride;
  const float* R;
  long long r_i_stride, r_o_stride, r_split_stride;
  const float* bias;
  const float* scale;
  int n_split;
  int I_out, O_out, N, Kc;
  int taps, tap_di, tap_do, o_mul, kchunks;
  int pre_act, post_act, i_tiles;
  int m_tiles, n_tiles;  // (I tiles x O_out) and N tiles
  int kpair;             // 1: 64-row tiles, promotion chunks alternating between the consumer warpgroups (host side)
};

template <int BN, int PREC>
struct TcCfg {
  static constexpr bool SPLIT = PREC == 0;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = TC_A_BYTES + B_BYTES * (SPLIT ? 2 : 1);
  static constexpr int STAGES = (200 * 1024 / STAGE_BYTES) > 8 ? 8 : (200 * 1024 / STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  // K-pair queue: a slot holds a 64 x BN fp32 chunk in Q_PIECES 8 KB pieces, piece h of slot q in the unused second half
  // of stage slot q * Q_PIECES + h's A tile
  static constexpr int Q_PIECES = BN / 32;
  static_assert(STAGES % 2 == 0 && 2 * Q_PIECES <= STAGES, "K-pair rings and queue");
};

// round-to-nearest (ties away) TF32 on the integer pipe: add half an ulp of the 10-bit mantissa to
// the magnitude bits and clear the low 13 bits (cvt.rna.tf32.f32 gives the same value but runs at
// the slow conversion rate).  |x - hi| <= 2^-12 |x|, so with lo = rna(x - hi) the split
// x ~ hi + lo is good to 2^-24 |x|: fp32-equivalent products.
// A NaN is quieted instead: the add would carry its payload into the exponent or the sign (0x7FFFFFFF, the NaN CUDA
// arithmetic returns, would become -0 and 0x7F800001 +Inf), and the tensor core reads only the top 19 bits.  Finite x
// with |x| >= 0x7F7FF000 (about 3.4e38) rounds to Inf, as rna does.
__device__ __forceinline__ float tf32_rna(float x) {
  const uint32_t u = __float_as_uint(x);
  return __uint_as_float((x != x ? u | 0x00400000u : u + 0x1000u) & 0xFFFFE000u);
}
// lo = rna(x - hi).  x - hi is NaN only for x = +-Inf or NaN, where hi alone carries the value: lo = 0.
__device__ __forceinline__ float tf32_rna_lo(float x, float hi) {
  const float d = x - hi;
  return d != d ? 0.f : __uint_as_float((__float_as_uint(d) + 0x1000u) & 0xFFFFE000u);
}

// fused activation of the tensor-core path (ELU through ex2.approx, common.cuh)
__device__ __forceinline__ float act_tc(float x, int act) {
  if (act == ACT_ELU) return elu_fast(x);
  if (act == ACT_GELU) return gelu_f(x);
  return x;
}

// The register-A fragments of one 32-wide K stage: thread (gq, tq) of its warp reads rows r0 and r0 + 8, columns tq and
// tq + 4 of every 8-wide K step out of a swizzled [128][32] fp32 tile at shared address `st` (a_row, a_sw: see the
// consumer below), applies the pre-activation and splits (SPLIT) or rounds each value.
// PRE_ELU: the fused pre-activation (ELU or none) is a template parameter and evaluated branch-free, so the consumer
// path from one wgmma group to the next has no data-dependent divergence (ptxas would otherwise serialise the wgmmas
// behind compiler-inserted warpgroup arrives).
template <bool SPLIT, bool PRE_ELU>
__device__ __forceinline__ void tc_build_a(uint32_t st, uint32_t a_row, uint32_t a_sw, uint32_t (&ah)[4][4], uint32_t (&al)[4][4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {   // a[e]: row r0 + 8 (e & 1), column 8 k + tq + 4 (e >> 1)
      const uint32_t chunk = (uint32_t)(2 * k + (e >> 1));
      float v;
      asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(st + a_row + (e & 1) * 1024u + ((chunk ^ a_sw) << 4)));
      if (PRE_ELU) {   // elu_fast, as a select: x > 0 ? x : exp(x) - 1
        const float e = __expf(v) - 1.f;
        v = v > 0.f ? v : e;
      }
      if (SPLIT) {
        // A non-finite x enters as (hi, lo) = (0, x - 0): the subtraction returns +-Inf or the canonical quiet NaN
        // 0x7FFFFFFF, which the mask keeps (no rounding add for it).  (hi, lo) = (Inf, 0) would make a_hi * b_lo
        // add Inf * w_lo, which is NaN for w_lo == 0 and for w_lo of the other sign, where x * w is +-Inf.
        // Finite x: the rna split above, bit for bit.
        const bool nonfinite = !(fabsf(v) < INFINITY);
        const float h = nonfinite ? 0.f : __uint_as_float((__float_as_uint(v) + 0x1000u) & 0xFFFFE000u);
        const float d = v - h;
        ah[k][e] = __float_as_uint(h);
        al[k][e] = (__float_as_uint(d) + (nonfinite ? 0u : 0x1000u)) & 0xFFFFE000u;
      } else {
        ah[k][e] = __float_as_uint(tf32_rna(v));
      }
    }
  }
}

// The wgmmas of one K stage: a_hi * b_hi into d0; a_lo * b_hi + a_hi * b_lo into d1 (SPLIT).  first: the stage starts
// fresh accumulators.
template <int BN, bool SPLIT>
__device__ __forceinline__ void tc_mma_stage(float (&d0)[BN / 2], float (&d1)[BN / 2], const uint32_t (&ah)[4][4],
                                             const uint32_t (&al)[4][4], uint64_t db, uint64_t dbl, bool first) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {   // 4 x (K = 8 tf32 = 32 bytes) per 128-byte row
    const uint32_t acc_in = (first && k == 0) ? 0u : 1u;
    wgmma_tf32_rs<BN>(d0, ah[k], db + (uint64_t)(2 * k), acc_in);                 // a_hi * b_hi
    if (SPLIT) {
      wgmma_tf32_rs<BN>(d1, al[k], db + (uint64_t)(2 * k), acc_in);               // a_lo * b_hi
      wgmma_tf32_rs<BN>(d1, ah[k], dbl + (uint64_t)(2 * k), 1u);                  // a_hi * b_lo
    }
  }
}

// KP: K-pair mode.  A template parameter, so that the 128-row form carries none of K-pair's branches (as a runtime flag
// they cost it about 10 %); the promotion adds and the epilogue are the same source in both forms, and
// tests/test_gemm_tc_kpair_gpu.py holds the two to equal bits.
template <int BN, int PREC, bool PRE_ELU, bool KP>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW,
               const __grid_constant__ CUtensorMap tmWlo, const TcParams p) {
  using Cfg = TcCfg<BN, PREC>;
  constexpr int S = Cfg::STAGES;
  constexpr int CH = TC_CHUNK_STAGES;
  constexpr int NR = BN / 2;   // accumulator registers per thread of a 64 x BN wgmma
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (128-byte swizzle atoms) as pointer arithmetic on the __shared__ array (an integer round trip
  // would demote every later access through `smem` to generic LD / ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S * Cfg::STAGE_BYTES);   // [S] TMA landed
  uint64_t* empty = full + S;                                                  // [S] every consumer warp reading it is done
  uint64_t* qfull = empty + S;                                                 // [2] K-pair: warpgroup 1's chunk is in the slot
  uint64_t* qempty = qfull + 2;                                                // [2] K-pair: warpgroup 0 has added it
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int total_k = p.taps * p.kchunks;
  const int total_tiles = p.m_tiles * p.n_tiles;
  const int bm = KP ? TC_BM / 2 : TC_BM;   // tile rows
  const int R = KP ? S / 2 : S;            // slots per ring: K-pair, slots [0, S/2) feed warpgroup 0, the rest 1

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], KP ? TC_CONSUMER_WARPS / 2 : TC_CONSUMER_WARPS);   // K-pair: one warpgroup reads a stage
    }
    for (int q = 0; q < 2; ++q) {
      mbar_init(&qfull[q], 128);
      mbar_init(&qempty[q], 128);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == TC_CONSUMER_WARPS) {
    // ================= TMA producer: one elected lane walks this CTA's stages (all its tiles back to back)
    if (elect_one()) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmW);
      if (Cfg::SPLIT) tma_prefetch_desc(&tmWlo);
      int pos0 = 0, ph0 = 0, pos1 = 0, ph1 = 0;   // next slot and its phase parity, per ring
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int nt = t % p.n_tiles, mt = t / p.n_tiles;
        const int i0 = (mt % p.i_tiles) * bm, ot = mt / p.i_tiles, n0 = nt * BN;
        for (int kit = 0; kit < total_k; ++kit) {
          const int w = KP ? (kit / TC_CHUNK_STAGES) & 1 : 0;   // the ring of the warpgroup that reads the stage
          const int pos = w ? pos1 : pos0, ph = w ? ph1 : ph0;
          const int s = w * R + pos;
          const int npos = pos + 1 == R ? 0 : pos + 1, nph = ph ^ (npos == 0);
          if (w) { pos1 = npos; ph1 = nph; } else { pos0 = npos; ph0 = nph; }
          mbar_wait(&empty[s], ph ^ 1);
          const int tap = kit / p.kchunks, kc = kit % p.kchunks;
          uint8_t* st = smem + s * Cfg::STAGE_BYTES;
          // the A box is bm rows (the plan's tensor map); in K-pair mode the slot's second 64 A rows stay unused
          mbar_arrive_expect_tx(&full[s], Cfg::STAGE_BYTES - (TC_BM - bm) * 128);
          tma_load_3d(st, &tmA, &full[s], kc * TC_BKE, i0 + tap * p.tap_di, ot * p.o_mul + tap * p.tap_do);
          tma_load_2d(st + TC_A_BYTES, &tmW, &full[s], kit * TC_BKE, n0);   // tap * Kc + kc * 32 == kit * 32
          if (Cfg::SPLIT) tma_load_2d(st + TC_A_BYTES + Cfg::B_BYTES, &tmWlo, &full[s], kit * TC_BKE, n0);
        }
      }
    }
    return;
  }

  // ================= consumers.  Thread (warp wq of warpgroup wg, lane = 4 gq + tq) holds A rows r0 and r0 + 8 of the
  // tile, columns tq and tq + 4 of every 8-wide K step (the wgmma register fragment); the accumulator fragment covers the
  // same two rows, columns 8 b + 2 tq and 8 b + 2 tq + 1 of every 8-column block b.  In K-pair mode both warpgroups
  // hold rows 0..63, so thread t of warpgroup 1 holds the accumulator elements of thread t of warpgroup 0.
  const int wg = warp / 4, wq = warp % 4, gq = lane / 4, tq = lane % 4;
  const int r0 = (KP ? 0 : wg * 64) + wq * 16 + gq;
  // element (r, c) of a stage's swizzled [128][32] fp32 A tile sits at byte r * 128 + ((c / 4) ^ (r % 8)) * 16 + (c % 4) * 4;
  // rows r0 and r0 + 8 share r % 8
  const uint32_t a_row = (uint32_t)r0 * 128u + (uint32_t)tq * 4u, a_sw = (uint32_t)(r0 & 7);
  const uint32_t smem0 = smem_u32(smem);
  float acc[NR], d0[NR], d1[NR];
#pragma unroll
  for (int j = 0; j < NR; ++j) d0[j] = d1[j] = 0.f;
  const int nch = (total_k + CH - 1) / CH;
  const bool sender = KP && wg == 1;   // K-pair: this warpgroup's chunks go through the queue
  // this thread's element j of queue slot q: 8 KB pieces of 16 x 128 fp32, element j * 128 + (thread in warpgroup)
  auto qel = [&](int q, int j) {
    return reinterpret_cast<float*>(smem + (q * Cfg::Q_PIECES + j / 16) * Cfg::STAGE_BYTES + TC_A_BYTES / 2) +
           (j % 16) * 128 + (threadIdx.x & 127);
  };
  int qn = 0;                               // chunks queued so far (slot qn & 1, use qn >> 1 of it)
  // warpgroup 0 adds the chunk warpgroup 1 queued, as acc += (d0 + d1) of that chunk
  auto take_queued = [&]() {
    mbar_wait(&qfull[qn & 1], (qn >> 1) & 1);
#pragma unroll
    for (int j = 0; j < NR; ++j) acc[j] += *qel(qn & 1, j);
    mbar_arrive(&qempty[qn & 1]);
    ++qn;
  };
  // this warpgroup's ring: every stage in the 128-row mode, its own chunks' stages in K-pair mode
  const int base = KP ? wg * R : 0;
  int pos = 0, ph = 0;
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const int nt = t % p.n_tiles, mt = t / p.n_tiles;
    const int i0 = (mt % p.i_tiles) * bm, ot = mt / p.i_tiles, n0 = nt * BN;
#pragma unroll
    for (int j = 0; j < NR; ++j) acc[j] = 0.f;
    // K in chunks of up to CH stages, each chunk's accumulators promoted after it.  Every wgmma wait sits outside any
    // branch, so ptxas needs no serialising warpgroup waits of its own.  The two consumer warpgroups overlap each other:
    // one builds fragments while the other's wgmmas run.
    for (int c = KP ? wg : 0; c < nch; c += KP ? 2 : 1) {
      const int k0 = c * CH;
      const int nst = total_k - k0 < CH ? total_k - k0 : CH;
      for (int u = 0; u < nst; ++u) {
        const int s = base + pos;
        mbar_wait(&full[s], ph);
        const uint32_t st = smem0 + (uint32_t)(s * Cfg::STAGE_BYTES);
        uint32_t ah[4][4], al[4][4];
        tc_build_a<Cfg::SPLIT, PRE_ELU>(st, a_row, a_sw, ah, al);
        const uint64_t db = gmma_desc_sw128(st + TC_A_BYTES);
        const uint64_t dbl = gmma_desc_sw128(st + TC_A_BYTES + Cfg::B_BYTES);
        wgmma_fence();
        tc_mma_stage<BN, Cfg::SPLIT>(d0, d1, ah, al, db, dbl, u == 0);   // a chunk starts fresh accumulators
        wgmma_commit();
        // the group's A operand is registers the next stage's fragments would overwrite: it must retire first
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);   // this warp's wgmmas have read the stage
        pos = pos + 1 == R ? 0 : pos + 1;
        ph ^= pos == 0;
      }
      fence_acc(d0);
      if (Cfg::SPLIT) fence_acc(d1);
      if (sender) {
        mbar_wait(&qempty[qn & 1], ((qn >> 1) & 1) ^ 1);
#pragma unroll
        for (int j = 0; j < NR; ++j) *qel(qn & 1, j) = Cfg::SPLIT ? d0[j] + d1[j] : d0[j];
        mbar_arrive(&qfull[qn & 1]);
        ++qn;
      } else {
        if (KP && c > 0) take_queued();   // chunk c - 1 first
#pragma unroll
        for (int j = 0; j < NR; ++j) acc[j] += Cfg::SPLIT ? d0[j] + d1[j] : d0[j];
      }
    }
    if (KP && !sender && nch % 2 == 0) take_queued();   // the tile's last chunk is warpgroup 1's
    if (sender) continue;   // warpgroup 0 writes the tile
    // ---- epilogue: bias, LayerScale, residual, activation -> global (8-byte stores: 4 lanes = one 32-byte sector)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int i = i0 + r0 + 8 * h;
      if (i >= p.I_out) continue;
      float* crow = p.C + (long long)ot * p.c_o_stride + (long long)i * p.c_i_stride;
      float* crow2 = p.C2 ? p.C2 + (long long)ot * p.c_o_stride + (long long)i * p.c_i_stride : nullptr;
      const float* rrow = p.R ? p.R + (long long)ot * p.r_o_stride + (long long)i * p.r_i_stride : nullptr;
#pragma unroll
      for (int b = 0; b < BN / 8; ++b) {
        const int n = n0 + 8 * b + 2 * tq;
        if (n < p.N) {   // N % 4 == 0: n + 1 < N as well
          float2 v = make_float2(acc[4 * b + 2 * h], acc[4 * b + 2 * h + 1]);
          if (p.bias) {
            const float2 bb = *reinterpret_cast<const float2*>(p.bias + n);
            v.x += bb.x; v.y += bb.y;
          }
          if (p.scale) {
            const float2 ss = *reinterpret_cast<const float2*>(p.scale + n);
            v.x *= ss.x; v.y *= ss.y;
          }
          long long coff = n, roff = n;
          if (p.n_split > 0) {   // n_split % 4 == 0: n and n + 1 fall in the same split
            const int j = n / p.n_split, co = n % p.n_split;
            coff = (long long)j * p.c_split_stride + co;
            roff = (long long)j * p.r_split_stride + co;
          }
          if (rrow) {
            const float2 rr = *reinterpret_cast<const float2*>(rrow + roff);
            v.x += rr.x; v.y += rr.y;
          }
          if (crow2)   // e.g. the ELU'd copy a resblock's first conv consumes while the skip reads the raw one
            *reinterpret_cast<float2*>(crow2 + coff) = make_float2(act_tc(v.x, p.act2), act_tc(v.y, p.act2));
          *reinterpret_cast<float2*>(crow + coff) = make_float2(act_tc(v.x, p.post_act), act_tc(v.y, p.post_act));
        }
      }
    }
  }
}

// ---------------------------------------------------------------- fused SEANet residual block (C = 64 or 128)
//   h = ELU(b1 + conv_k3(ELU(y)))   (C -> C/2, causal: output step t reads y rows t-2, t-1, t)
//   r = ELU(y + b2 + W2 h)          (1x1, C/2 -> C)
// in one persistent launch at precision 0, with the same operations in the same order as the two gemm_tc launches it
// replaces.  A tile is 128 streams at one time step.  Phase 1 is gemm_tc's K loop over 3 taps x C/32 stages of raw y
// (ELU in the fragment build) against W1 (N = C/2); its epilogue writes h into shared memory as [128][32] swizzled
// blocks, the layout the fragment builder reads.  Phase 2 takes A = h from there and B = W2 from the ring, one stage per
// 64-column N slice (both K stages of the slice in it).  The residual y[t] is the A tile of phase 1's tap-2 stages: the
// consumers keep those ring slots until the slice's epilogue has read them, so y is read from HBM once and the hidden
// tensor never leaves the SM.
constexpr int RB_B_BYTES = 64 * 128;                         // one W stage of up to 64 rows x 32 fp32
constexpr int RB_STAGE_BYTES = TC_A_BYTES + 2 * RB_B_BYTES;  // 32 KB: [y 128 x 32 | W hi | W lo]
constexpr int RB_STAGES = 6;

struct RbParams {
  float* out;
  long long o_i_stride, o_o_stride;
  const float* b1;
  const float* b2;
  int I_out, i_tiles, m_tiles;
};

template <int C>
struct RbCfg {
  static constexpr int N1 = C / 2;         // hidden width
  static constexpr int KCH = C / 32;       // phase-1 stages per tap
  static constexpr int P1 = 3 * KCH;       // phase-1 stages
  static constexpr int NS = C / 64;        // phase-2 N slices (one ring stage each)
  static constexpr int K2 = N1 / 32;       // phase-2 K stages per slice
  static constexpr int H_BYTES = K2 * TC_A_BYTES;
  static constexpr int SMEM_BYTES = RB_STAGES * RB_STAGE_BYTES + H_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  // phase 2's stages must not land on the slots still held for the residual (else the producer would wait on the
  // consumers, which wait on it)
  static constexpr bool ring_ok() {
    for (int j = 0; j < NS; ++j)
      for (int kc = 0; kc < KCH; ++kc)
        if ((P1 + j) % RB_STAGES == (2 * KCH + kc) % RB_STAGES) return false;
    return RB_STAGES >= KCH + NS;
  }
  static_assert(ring_ok(), "ring too small for the held residual stages");
  static_assert(K2 * 2 * RB_B_BYTES <= RB_STAGE_BYTES, "a phase-2 slice must fit one stage");
};

template <int C>
__global__ void __launch_bounds__(TC_THREADS, 1)
resblock_tc_kernel(const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmW1,
                   const __grid_constant__ CUtensorMap tmW1lo, const __grid_constant__ CUtensorMap tmW2,
                   const __grid_constant__ CUtensorMap tmW2lo, const RbParams p) {
  using Cfg = RbCfg<C>;
  constexpr int S = RB_STAGES;
  constexpr int CH = TC_CHUNK_STAGES;
  constexpr int N1 = Cfg::N1, NR1 = N1 / 2, KCH = Cfg::KCH, P1 = Cfg::P1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* hs = smem + S * RB_STAGE_BYTES;                     // h: K2 blocks of [128][32] fp32, 128-byte swizzle
  uint64_t* full = reinterpret_cast<uint64_t*>(hs + Cfg::H_BYTES);
  uint64_t* empty = full + S;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], TC_CONSUMER_WARPS);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == TC_CONSUMER_WARPS) {
    // ================= TMA producer
    if (elect_one()) {
      tma_prefetch_desc(&tmY);
      tma_prefetch_desc(&tmW1);
      tma_prefetch_desc(&tmW1lo);
      tma_prefetch_desc(&tmW2);
      tma_prefetch_desc(&tmW2lo);
      int g = 0;
      for (int t = blockIdx.x; t < p.m_tiles; t += gridDim.x) {
        const int i0 = (t % p.i_tiles) * TC_BM, ot = t / p.i_tiles;
        for (int kit = 0; kit < P1; ++kit, ++g) {
          const int s = g % S;
          mbar_wait(&empty[s], ((g / S) & 1) ^ 1);
          const int tap = kit / KCH, kc = kit % KCH;
          uint8_t* st = smem + s * RB_STAGE_BYTES;
          mbar_arrive_expect_tx(&full[s], TC_A_BYTES + 2 * N1 * 128);
          tma_load_3d(st, &tmY, &full[s], kc * TC_BKE, i0, ot + tap);
          tma_load_2d(st + TC_A_BYTES, &tmW1, &full[s], kit * TC_BKE, 0);
          tma_load_2d(st + TC_A_BYTES + RB_B_BYTES, &tmW1lo, &full[s], kit * TC_BKE, 0);
        }
        for (int ns = 0; ns < Cfg::NS; ++ns, ++g) {
          const int s = g % S;
          mbar_wait(&empty[s], ((g / S) & 1) ^ 1);
          uint8_t* st = smem + s * RB_STAGE_BYTES;
          mbar_arrive_expect_tx(&full[s], Cfg::K2 * 2 * RB_B_BYTES);
#pragma unroll
          for (int kc = 0; kc < Cfg::K2; ++kc) {   // [W2 hi k0 | W2 lo k0 | W2 hi k1 | W2 lo k1]
            tma_load_2d(st + kc * 2 * RB_B_BYTES, &tmW2, &full[s], kc * TC_BKE, ns * 64);
            tma_load_2d(st + kc * 2 * RB_B_BYTES + RB_B_BYTES, &tmW2lo, &full[s], kc * TC_BKE, ns * 64);
          }
        }
      }
    }
    return;
  }

  // ================= consumers (fragment ownership as in gemm_tc_kernel)
  const int wg = warp / 4, wq = warp % 4, gq = lane / 4, tq = lane % 4;
  const int r0 = wg * 64 + wq * 16 + gq;
  const uint32_t a_row = (uint32_t)r0 * 128u + (uint32_t)tq * 4u, a_sw = (uint32_t)(r0 & 7);
  const uint32_t smem0 = smem_u32(smem), hs0 = smem_u32(hs);
  int g = 0;
  for (int t = blockIdx.x; t < p.m_tiles; t += gridDim.x) {
    const int i0 = (t % p.i_tiles) * TC_BM, ot = t / p.i_tiles;
    const int g_res = g + 2 * KCH;   // ring index of the first tap-2 stage: y[t], channels 0..31
    {
      // ---- phase 1: k3 conv C -> C/2 over ELU(y), promoted every CH stages
      float acc[NR1], d0[NR1], d1[NR1];
#pragma unroll
      for (int j = 0; j < NR1; ++j) acc[j] = d0[j] = d1[j] = 0.f;
      for (int k0 = 0; k0 < P1; k0 += CH) {
        const int nst = P1 - k0 < CH ? P1 - k0 : CH;
        for (int u = 0; u < nst; ++u, ++g) {
          const int s = g % S;
          mbar_wait(&full[s], (g / S) & 1);
          const uint32_t st = smem0 + (uint32_t)(s * RB_STAGE_BYTES);
          uint32_t ah[4][4], al[4][4];
          tc_build_a<true, true>(st, a_row, a_sw, ah, al);
          wgmma_fence();
          tc_mma_stage<N1, true>(d0, d1, ah, al, gmma_desc_sw128(st + TC_A_BYTES), gmma_desc_sw128(st + TC_A_BYTES + RB_B_BYTES),
                                 u == 0);
          wgmma_commit();
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0 && k0 + u < 2 * KCH) mbar_arrive(&empty[s]);   // tap-2 stages stay until the residual is read
        }
        fence_acc(d0);
        fence_acc(d1);
#pragma unroll
        for (int j = 0; j < NR1; ++j) acc[j] += d0[j] + d1[j];
      }
      // ---- h = ELU(acc + b1) -> shared memory.  Each warpgroup writes and reads only its own 64 rows: the barrier
      // before the write waits for the warpgroup's phase-2 reads of the previous tile, the one after publishes h.
      named_bar_sync(1 + wg, 128);
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = r0 + 8 * hh;
#pragma unroll
        for (int b = 0; b < N1 / 8; ++b) {
          const int n = 8 * b + 2 * tq;
          const float2 bb = *reinterpret_cast<const float2*>(p.b1 + n);
          float2 v = make_float2(acc[4 * b + 2 * hh], acc[4 * b + 2 * hh + 1]);
          v.x += bb.x; v.y += bb.y;
          const uint32_t cc = (uint32_t)(n % 32);
          const uint32_t addr = hs0 + (uint32_t)(n / 32) * TC_A_BYTES + (uint32_t)r * 128u + (((cc >> 2) ^ (uint32_t)(r & 7)) << 4) +
                                (cc & 3u) * 4u;
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(act_tc(v.x, ACT_ELU)), "f"(act_tc(v.y, ACT_ELU))
                       : "memory");
        }
      }
      named_bar_sync(1 + wg, 128);
    }
    // ---- phase 2: 1x1 conv C/2 -> C, one 64-column slice at a time; epilogue + residual + ELU -> global
    for (int ns = 0; ns < Cfg::NS; ++ns, ++g) {
      const int s = g % S;
      mbar_wait(&full[s], (g / S) & 1);
      const uint32_t st = smem0 + (uint32_t)(s * RB_STAGE_BYTES);
      float acc[32], d0[32], d1[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) d0[j] = d1[j] = 0.f;
#pragma unroll
      for (int kc = 0; kc < Cfg::K2; ++kc) {
        uint32_t ah[4][4], al[4][4];
        tc_build_a<true, false>(hs0 + (uint32_t)(kc * TC_A_BYTES), a_row, a_sw, ah, al);
        const uint32_t wst = st + (uint32_t)(kc * 2 * RB_B_BYTES);
        wgmma_fence();
        tc_mma_stage<64, true>(d0, d1, ah, al, gmma_desc_sw128(wst), gmma_desc_sw128(wst + RB_B_BYTES), kc == 0);
        wgmma_commit();
        wgmma_wait<0>();
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      fence_acc(d0);
      fence_acc(d1);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        acc[j] = 0.f;
        acc[j] += d0[j] + d1[j];
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = r0 + 8 * hh;
        const int i = i0 + r;
        if (i >= p.I_out) continue;
        float* orow = p.out + (long long)ot * p.o_o_stride + (long long)i * p.o_i_stride;
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          const int n = ns * 64 + 8 * b + 2 * tq;
          const float2 bb = *reinterpret_cast<const float2*>(p.b2 + n);
          float2 v = make_float2(acc[4 * b + 2 * hh], acc[4 * b + 2 * hh + 1]);
          v.x += bb.x; v.y += bb.y;
          const uint32_t cc = (uint32_t)(n % 32);
          const int rs = (g_res + n / 32) % S;   // the tap-2 stage holding y[t], channels n / 32 * 32 ...
          const float2 rr = *reinterpret_cast<const float2*>(smem + rs * RB_STAGE_BYTES + r * 128 +
                                                             (((cc >> 2) ^ (uint32_t)(r & 7)) << 4) + (cc & 3u) * 4u);
          v.x += rr.x; v.y += rr.y;
          *reinterpret_cast<float2*>(orow + n) = make_float2(act_tc(v.x, ACT_ELU), act_tc(v.y, ACT_ELU));
        }
      }
      __syncwarp();
      if (lane == 0) {   // this slice's residual stages are read
        mbar_arrive(&empty[(g_res + 2 * ns) % S]);
        mbar_arrive(&empty[(g_res + 2 * ns + 1) % S]);
      }
    }
  }
}

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && p) fn = (EncodeTiledFn)p;
  }
  return fn;
}

}  // namespace rstnet
using namespace rstnet;

struct rstnet_tc_plan {
  CUtensorMap tmA, tmW, tmWlo;
  TcParams p;
  dim3 grid;     // persistent CTAs: min(tiles, SMs)
  int bn, prec;
};

template <int BN, int PREC, bool PRE_ELU, bool KP>
static int tc_launch(const rstnet_tc_plan* pl, cudaStream_t st) {
  using Cfg = TcCfg<BN, PREC>;
  static unsigned long long attr = 0;
  smem_optin(gemm_tc_kernel<BN, PREC, PRE_ELU, KP>, Cfg::SMEM_BYTES, attr);
  gemm_tc_kernel<BN, PREC, PRE_ELU, KP><<<pl->grid, TC_THREADS, Cfg::SMEM_BYTES, st>>>(pl->tmA, pl->tmW, pl->tmWlo, pl->p);
  count_launch();
  return check_launch("gemm_tc");
}

template <int BN, int PREC>
static int tc_launch_mode(const rstnet_tc_plan* pl, cudaStream_t st) {
  const bool elu = pl->p.pre_act == ACT_ELU;
  if (pl->p.kpair) return elu ? tc_launch<BN, PREC, true, true>(pl, st) : tc_launch<BN, PREC, false, true>(pl, st);
  return elu ? tc_launch<BN, PREC, true, false>(pl, st) : tc_launch<BN, PREC, false, false>(pl, st);
}

extern "C" int rstnet_tc_gemm_create_ex(const rstnet_tc_gemm_desc* d, int32_t kpair, rstnet_tc_plan** out) {
  RSTNET_REQUIRE(d && out, "tc_gemm_create: null argument");
  RSTNET_REQUIRE(kpair >= -1 && kpair <= 1, "tc_gemm_create: kpair must be -1 (auto), 0 or 1 (got %d)", kpair);
  RSTNET_REQUIRE(d->A && d->W && d->C, "tc_gemm_create: null tensor pointer");
  RSTNET_REQUIRE(d->precision != 0 || d->W_lo, "tc_gemm_create: precision 0 (3xTF32) needs W_lo");
  RSTNET_REQUIRE(d->Kc > 0 && d->Kc % TC_BKE == 0, "tc_gemm_create: Kc (%d) must be a multiple of %d", d->Kc, TC_BKE);
  RSTNET_REQUIRE(d->N > 0 && d->N % 4 == 0, "tc_gemm_create: N (%d) must be a multiple of 4", d->N);
  RSTNET_REQUIRE(d->taps >= 1 && d->I_out > 0 && d->O_out > 0, "tc_gemm_create: bad shape");
  RSTNET_REQUIRE(d->precision == 0 || d->precision == 1, "tc_gemm_create: precision must be 0 (3xTF32) or 1 (TF32)");
  RSTNET_REQUIRE(d->pre_act == ACT_NONE || d->pre_act == ACT_ELU, "tc_gemm_create: pre_act must be NONE or ELU (got %d)", d->pre_act);
  RSTNET_REQUIRE((uintptr_t)d->A % 16 == 0 && (uintptr_t)d->W % 16 == 0 && (uintptr_t)d->C % 16 == 0 &&
                     d->a_i_stride % 4 == 0 && d->a_o_stride % 4 == 0 && d->c_i_stride % 4 == 0 && d->c_o_stride % 4 == 0 &&
                     d->c_split_stride % 4 == 0 && d->n_split % 4 == 0,
                 "tc_gemm_create: 16-byte alignment required");
  EncodeTiledFn enc = get_encode_fn();
  RSTNET_REQUIRE(enc != nullptr, "tc_gemm_create: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  rstnet_tc_plan* pl = new rstnet_tc_plan();
  const int N = d->N;
  const int sms = sm_count();
  pl->bn = N >= 64 ? 64 : 32;
  const int i_tiles = ceil_div(d->I_out, TC_BM);
  {
    // narrow the tile when that takes fewer rounds of the SMs (a BN=64 tile costs ~1.5x a BN=32 tile: same A fragment
    // loads and splits, twice the MMAs)
    const long long mt = (long long)i_tiles * d->O_out;
    const long long t64 = mt * ceil_div(N, 64), t32 = mt * ceil_div(N, 32);
    if (pl->bn == 64 && ((t32 + sms - 1) / sms) * 2 <= ((t64 + sms - 1) / sms) * 3) pl->bn = 32;
  }
  pl->prec = d->precision;
  const int n_tiles = ceil_div(N, pl->bn);
  if (kpair < 0) {
    // K-pair (64-row tiles, the promotion chunks split between the two consumer warpgroups) for the few-tile, long-K
    // launches: when the 128-row tiles fit in one round of the SMs and K-pair takes fewer rounds times serial K stages.
    // A tie keeps 128-row tiles.  Past one round the per-tile cost decides: at 3 840 tiles of K = 256 (the 12.5 kHz
    // decoder's transposed conv) the rule alone would pick K-pair, which ran 1.6x slower there.
    const long long total_k = (long long)d->taps * (d->Kc / TC_BKE);
    const long long t128 = (long long)i_tiles * d->O_out * n_tiles, t64 = (long long)ceil_div(d->I_out, TC_BM / 2) * d->O_out * n_tiles;
    const long long pair_k = (total_k + 2 * TC_CHUNK_STAGES - 1) / (2 * TC_CHUNK_STAGES) * TC_CHUNK_STAGES;
    kpair = t128 <= sms && ((t64 + sms - 1) / sms) * pair_k < total_k;
  }
  const int bm = kpair ? TC_BM / 2 : TC_BM;
  {
    cuuint64_t gdim[3] = {(cuuint64_t)d->a_c_extent, (cuuint64_t)d->a_i_extent, (cuuint64_t)d->a_o_extent};
    cuuint64_t gstr[2] = {(cuuint64_t)d->a_i_stride * 4, (cuuint64_t)d->a_o_stride * 4};
    cuuint32_t box[3] = {TC_BKE, (cuuint32_t)bm, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&pl->tmA, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)d->A, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      delete pl;
      set_error("tc_gemm_create: cuTensorMapEncodeTiled(A) failed with %d", (int)r);
      return 3;
    }
  }
  {
    cuuint64_t gdim[2] = {(cuuint64_t)d->taps * d->Kc, (cuuint64_t)N};
    cuuint64_t gstr[1] = {(cuuint64_t)d->taps * d->Kc * 4};
    cuuint32_t box[2] = {TC_BKE, (cuuint32_t)pl->bn};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&pl->tmW, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)d->W, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r == CUDA_SUCCESS && d->W_lo)
      r = enc(&pl->tmWlo, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)d->W_lo, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    else
      pl->tmWlo = pl->tmW;
    if (r != CUDA_SUCCESS) {
      delete pl;
      set_error("tc_gemm_create: cuTensorMapEncodeTiled(W) failed with %d", (int)r);
      return 3;
    }
  }
  TcParams& p = pl->p;
  p.C2 = d->C2; p.act2 = d->act2;
  p.C = d->C; p.c_i_stride = d->c_i_stride; p.c_o_stride = d->c_o_stride; p.c_split_stride = d->c_split_stride;
  p.R = d->R; p.r_i_stride = d->r_i_stride; p.r_o_stride = d->r_o_stride; p.r_split_stride = d->r_split_stride;
  p.bias = d->bias; p.scale = d->scale; p.n_split = d->n_split;
  p.I_out = d->I_out; p.O_out = d->O_out; p.N = N; p.Kc = d->Kc;
  p.taps = d->taps; p.tap_di = d->tap_di; p.tap_do = d->tap_do; p.o_mul = d->o_mul; p.kchunks = d->Kc / TC_BKE;
  p.pre_act = d->pre_act; p.post_act = d->post_act;
  p.kpair = kpair;
  p.i_tiles = ceil_div(d->I_out, bm);
  p.m_tiles = p.i_tiles * d->O_out;
  p.n_tiles = n_tiles;
  const long long tiles = (long long)p.m_tiles * p.n_tiles;
  pl->grid = dim3((unsigned)(tiles < sms ? tiles : sms));
  *out = pl;
  return 0;
}

extern "C" int rstnet_tc_gemm_create(const rstnet_tc_gemm_desc* d, rstnet_tc_plan** out) {
  return rstnet_tc_gemm_create_ex(d, -1, out);
}

extern "C" int rstnet_tc_gemm_run(const rstnet_tc_plan* pl, rstnet_stream_t stream) {
  RSTNET_REQUIRE(pl != nullptr, "tc_gemm_run: null plan");
  cudaStream_t st = (cudaStream_t)stream;
  if (pl->prec == 0) return pl->bn == 64 ? tc_launch_mode<64, 0>(pl, st) : tc_launch_mode<32, 0>(pl, st);
  return pl->bn == 64 ? tc_launch_mode<64, 1>(pl, st) : tc_launch_mode<32, 1>(pl, st);
}

extern "C" void rstnet_tc_gemm_destroy(rstnet_tc_plan* pl) { delete pl; }

struct rstnet_tc_resblock_plan {
  CUtensorMap tmY, tmW1, tmW1lo, tmW2, tmW2lo;
  RbParams p;
  dim3 grid;
  int channels;
};

static int encode_2d(CUtensorMap* m, const float* base, int cols, int rows, int box_rows) {
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstr[1] = {(cuuint64_t)cols * 4};
  cuuint32_t box[2] = {TC_BKE, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return (int)get_encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

extern "C" int rstnet_tc_resblock_create(const rstnet_tc_resblock_desc* d, rstnet_tc_resblock_plan** out) {
  RSTNET_REQUIRE(d && out, "tc_resblock_create: null argument");
  RSTNET_REQUIRE(d->Y && d->W1 && d->W1_lo && d->b1 && d->W2 && d->W2_lo && d->b2 && d->out, "tc_resblock_create: null pointer");
  const int Cc = d->channels;
  RSTNET_REQUIRE(Cc == 64 || Cc == 128, "tc_resblock_create: channels must be 64 or 128 (got %d)", Cc);
  RSTNET_REQUIRE(d->I_out > 0 && d->O_out > 0 && d->y_rows >= d->O_out + 2, "tc_resblock_create: bad shape");
  RSTNET_REQUIRE((uintptr_t)d->Y % 16 == 0 && (uintptr_t)d->W1 % 16 == 0 && (uintptr_t)d->W1_lo % 16 == 0 && (uintptr_t)d->W2 % 16 == 0 &&
                     (uintptr_t)d->W2_lo % 16 == 0 && (uintptr_t)d->out % 16 == 0 && (uintptr_t)d->b1 % 8 == 0 &&
                     (uintptr_t)d->b2 % 8 == 0 && d->y_i_stride % 4 == 0 && d->y_o_stride % 4 == 0 && d->out_i_stride % 4 == 0 &&
                     d->out_o_stride % 4 == 0,
                 "tc_resblock_create: 16-byte alignment required");
  RSTNET_REQUIRE(get_encode_fn() != nullptr, "tc_resblock_create: cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  rstnet_tc_resblock_plan* pl = new rstnet_tc_resblock_plan();
  pl->channels = Cc;
  int r;
  {
    cuuint64_t gdim[3] = {(cuuint64_t)Cc, (cuuint64_t)d->I_out, (cuuint64_t)d->y_rows};
    cuuint64_t gstr[2] = {(cuuint64_t)d->y_i_stride * 4, (cuuint64_t)d->y_o_stride * 4};
    cuuint32_t box[3] = {TC_BKE, TC_BM, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    r = (int)get_encode_fn()(&pl->tmY, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)d->Y, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r == CUDA_SUCCESS) r = encode_2d(&pl->tmW1, d->W1, 3 * Cc, Cc / 2, Cc / 2);
  if (r == CUDA_SUCCESS) r = encode_2d(&pl->tmW1lo, d->W1_lo, 3 * Cc, Cc / 2, Cc / 2);
  if (r == CUDA_SUCCESS) r = encode_2d(&pl->tmW2, d->W2, Cc / 2, Cc, 64);
  if (r == CUDA_SUCCESS) r = encode_2d(&pl->tmW2lo, d->W2_lo, Cc / 2, Cc, 64);
  if (r != CUDA_SUCCESS) {
    delete pl;
    set_error("tc_resblock_create: cuTensorMapEncodeTiled failed with %d", r);
    return 3;
  }
  RbParams& p = pl->p;
  p.out = d->out; p.o_i_stride = d->out_i_stride; p.o_o_stride = d->out_o_stride;
  p.b1 = d->b1; p.b2 = d->b2;
  p.I_out = d->I_out;
  p.i_tiles = ceil_div(d->I_out, TC_BM);
  p.m_tiles = p.i_tiles * d->O_out;
  const int sms = sm_count();
  pl->grid = dim3((unsigned)(p.m_tiles < sms ? p.m_tiles : sms));
  *out = pl;
  return 0;
}

template <int Cc>
static int rb_launch(const rstnet_tc_resblock_plan* pl, cudaStream_t st) {
  constexpr int smem = RbCfg<Cc>::SMEM_BYTES;
  static unsigned long long attr = 0;
  smem_optin(resblock_tc_kernel<Cc>, smem, attr);
  resblock_tc_kernel<Cc><<<pl->grid, TC_THREADS, smem, st>>>(pl->tmY, pl->tmW1, pl->tmW1lo, pl->tmW2, pl->tmW2lo, pl->p);
  count_launch();
  return check_launch("tc_resblock");
}

extern "C" int rstnet_tc_resblock_run(const rstnet_tc_resblock_plan* pl, rstnet_stream_t stream) {
  RSTNET_REQUIRE(pl != nullptr, "tc_resblock_run: null plan");
  cudaStream_t st = (cudaStream_t)stream;
  return pl->channels == 64 ? rb_launch<64>(pl, st) : rb_launch<128>(pl, st);
}

extern "C" void rstnet_tc_resblock_destroy(rstnet_tc_resblock_plan* pl) { delete pl; }
extern "C" int rstnet_tc_gemm_grid(const rstnet_tc_plan* pl, int32_t* gx, int32_t* gy, int32_t* bn) {
  if (!pl) return 1;
  *gx = ceil_div(pl->p.I_out, TC_BM) * pl->p.O_out; *gy = pl->p.n_tiles; *bn = pl->bn;
  return 0;
}
extern "C" int rstnet_tc_gemm_kpair(const rstnet_tc_plan* pl, int32_t* on) {
  if (!pl) return 1;
  *on = pl->p.kpair;
  return 0;
}

namespace rstnet {
__global__ void tf32_split_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i], h = tf32_rna(v);
    hi[i] = h;
    lo[i] = tf32_rna_lo(v, h);
  }
}
}  // namespace rstnet

extern "C" int rstnet_tf32_split_f32(const float* x, float* hi, float* lo, int64_t n, rstnet_stream_t stream) {
  RSTNET_REQUIRE(x && hi && lo, "tf32_split: null pointer");
  if (n <= 0) return 0;
  int g = ceil_div(n, 256);
  if (g > sm_count() * 8) g = sm_count() * 8;
  rstnet::tf32_split_kernel<<<g, 256, 0, (cudaStream_t)stream>>>(x, hi, lo, n);
  count_launch();
  return check_launch("tf32_split");
}
