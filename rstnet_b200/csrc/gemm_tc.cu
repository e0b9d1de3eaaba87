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
};

template <int BN, int PREC>
struct TcCfg {
  static constexpr bool SPLIT = PREC == 0;
  static constexpr int B_BYTES = BN * 128;
  static constexpr int STAGE_BYTES = TC_A_BYTES + B_BYTES * (SPLIT ? 2 : 1);
  static constexpr int STAGES = (200 * 1024 / STAGE_BYTES) > 8 ? 8 : (200 * 1024 / STAGE_BYTES);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

// round-to-nearest (ties away) TF32 on the integer pipe: add half an ulp of the 10-bit mantissa to
// the magnitude bits and clear the low 13 bits (cvt.rna.tf32.f32 gives the same value but runs at
// the slow conversion rate).  |x - hi| <= 2^-12 |x|, so with lo = rna(x - hi) the split
// x ~ hi + lo is good to 2^-24 |x|: fp32-equivalent products.
__device__ __forceinline__ float tf32_rna(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// fused activation of the tensor-core path (ELU through ex2.approx, common.cuh)
__device__ __forceinline__ float act_tc(float x, int act) {
  if (act == ACT_ELU) return elu_fast(x);
  if (act == ACT_GELU) return gelu_f(x);
  return x;
}

// PRE_ELU: the fused pre-activation (ELU or none) is a template parameter and evaluated branch-free, so the consumer
// path from one wgmma group to the next has no data-dependent divergence (ptxas would otherwise serialise the wgmmas
// behind compiler-inserted warpgroup arrives).
template <int BN, int PREC, bool PRE_ELU>
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
  uint64_t* empty = full + S;                                                  // [S] every consumer warp is done with it
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int total_k = p.taps * p.kchunks;
  const int total_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], TC_CONSUMER_WARPS);
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
      int g = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int nt = t % p.n_tiles, mt = t / p.n_tiles;
        const int i0 = (mt % p.i_tiles) * TC_BM, ot = mt / p.i_tiles, n0 = nt * BN;
        for (int kit = 0; kit < total_k; ++kit, ++g) {
          const int s = g % S;
          mbar_wait(&empty[s], ((g / S) & 1) ^ 1);
          const int tap = kit / p.kchunks, kc = kit % p.kchunks;
          uint8_t* st = smem + s * Cfg::STAGE_BYTES;
          mbar_arrive_expect_tx(&full[s], Cfg::STAGE_BYTES);
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
  // same two rows, columns 8 b + 2 tq and 8 b + 2 tq + 1 of every 8-column block b.
  const int wg = warp / 4, wq = warp % 4, gq = lane / 4, tq = lane % 4;
  const int r0 = wg * 64 + wq * 16 + gq;
  // element (r, c) of a stage's swizzled [128][32] fp32 A tile sits at byte r * 128 + ((c / 4) ^ (r % 8)) * 16 + (c % 4) * 4;
  // rows r0 and r0 + 8 share r % 8
  const uint32_t a_row = (uint32_t)r0 * 128u + (uint32_t)tq * 4u, a_sw = (uint32_t)(r0 & 7);
  const uint32_t smem0 = smem_u32(smem);
  float acc[NR], d0[NR], d1[NR];
#pragma unroll
  for (int j = 0; j < NR; ++j) d0[j] = d1[j] = 0.f;
  int g = 0;
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const int nt = t % p.n_tiles, mt = t / p.n_tiles;
    const int i0 = (mt % p.i_tiles) * TC_BM, ot = mt / p.i_tiles, n0 = nt * BN;
#pragma unroll
    for (int j = 0; j < NR; ++j) acc[j] = 0.f;
    // K in chunks of up to CH stages, each chunk's accumulators promoted after it.  Every wgmma wait sits outside any
    // branch, so ptxas needs no serialising warpgroup waits of its own.  The two consumer warpgroups overlap each other:
    // one builds fragments while the other's wgmmas run.
    for (int k0 = 0; k0 < total_k; k0 += CH) {
      const int nst = total_k - k0 < CH ? total_k - k0 : CH;
      for (int u = 0; u < nst; ++u, ++g) {
        const int s = g % S;
        mbar_wait(&full[s], (g / S) & 1);
        const uint32_t st = smem0 + (uint32_t)(s * Cfg::STAGE_BYTES);
        uint32_t ah[4][4], al[4][4];
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
            const float h = tf32_rna(v);
            ah[k][e] = __float_as_uint(h);
            al[k][e] = __float_as_uint(tf32_rna(v - h));
          }
        }
        const uint64_t db = gmma_desc_sw128(st + TC_A_BYTES);
        const uint64_t dbl = gmma_desc_sw128(st + TC_A_BYTES + Cfg::B_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // 4 x (K = 8 tf32 = 32 bytes) per 128-byte row
          const uint32_t acc_in = (u == 0 && k == 0) ? 0u : 1u;   // a chunk starts fresh accumulators
          wgmma_tf32_rs<BN>(d0, ah[k], db + (uint64_t)(2 * k), acc_in);                 // a_hi * b_hi
          if (Cfg::SPLIT) {
            wgmma_tf32_rs<BN>(d1, al[k], db + (uint64_t)(2 * k), acc_in);               // a_lo * b_hi
            wgmma_tf32_rs<BN>(d1, ah[k], dbl + (uint64_t)(2 * k), 1u);                  // a_hi * b_lo
          }
        }
        wgmma_commit();
        // the group's A operand is registers the next stage's fragments would overwrite: it must retire first
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);   // this warp's wgmmas have read the stage
      }
      fence_acc(d0);
      if (Cfg::SPLIT) fence_acc(d1);
#pragma unroll
      for (int j = 0; j < NR; ++j) acc[j] += Cfg::SPLIT ? d0[j] + d1[j] : d0[j];
    }
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

template <int BN, int PREC, bool PRE_ELU>
static int tc_launch(const rstnet_tc_plan* pl, cudaStream_t st) {
  using Cfg = TcCfg<BN, PREC>;
  static unsigned long long attr = 0;
  smem_optin(gemm_tc_kernel<BN, PREC, PRE_ELU>, Cfg::SMEM_BYTES, attr);
  gemm_tc_kernel<BN, PREC, PRE_ELU><<<pl->grid, TC_THREADS, Cfg::SMEM_BYTES, st>>>(pl->tmA, pl->tmW, pl->tmWlo, pl->p);
  count_launch();
  return check_launch("gemm_tc");
}

extern "C" int rstnet_tc_gemm_create(const rstnet_tc_gemm_desc* d, rstnet_tc_plan** out) {
  RSTNET_REQUIRE(d && out, "tc_gemm_create: null argument");
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
  {
    cuuint64_t gdim[3] = {(cuuint64_t)d->a_c_extent, (cuuint64_t)d->a_i_extent, (cuuint64_t)d->a_o_extent};
    cuuint64_t gstr[2] = {(cuuint64_t)d->a_i_stride * 4, (cuuint64_t)d->a_o_stride * 4};
    cuuint32_t box[3] = {TC_BKE, TC_BM, 1};
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
  p.pre_act = d->pre_act; p.post_act = d->post_act; p.i_tiles = i_tiles;
  p.m_tiles = i_tiles * d->O_out;
  p.n_tiles = ceil_div(N, pl->bn);
  const long long tiles = (long long)p.m_tiles * p.n_tiles;
  pl->grid = dim3((unsigned)(tiles < sms ? tiles : sms));
  *out = pl;
  return 0;
}

extern "C" int rstnet_tc_gemm_run(const rstnet_tc_plan* pl, rstnet_stream_t stream) {
  RSTNET_REQUIRE(pl != nullptr, "tc_gemm_run: null plan");
  cudaStream_t st = (cudaStream_t)stream;
  const bool elu = pl->p.pre_act == ACT_ELU;
  if (pl->prec == 0) {
    if (pl->bn == 64) return elu ? tc_launch<64, 0, true>(pl, st) : tc_launch<64, 0, false>(pl, st);
    return elu ? tc_launch<32, 0, true>(pl, st) : tc_launch<32, 0, false>(pl, st);
  }
  if (pl->bn == 64) return elu ? tc_launch<64, 1, true>(pl, st) : tc_launch<64, 1, false>(pl, st);
  return elu ? tc_launch<32, 1, true>(pl, st) : tc_launch<32, 1, false>(pl, st);
}

extern "C" void rstnet_tc_gemm_destroy(rstnet_tc_plan* pl) { delete pl; }
extern "C" int rstnet_tc_gemm_grid(const rstnet_tc_plan* pl, int32_t* gx, int32_t* gy, int32_t* bn) {
  if (!pl) return 1;
  *gx = pl->p.m_tiles; *gy = pl->p.n_tiles; *bn = pl->bn;
  return 0;
}

namespace rstnet {
__global__ void tf32_split_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i], h = tf32_rna(v);
    hi[i] = h;
    lo[i] = tf32_rna(v - h);
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
