// Weight-streaming skinny GEMM for the LM decode step (wgmma, bf16 operands, fp32 accumulate in
// registers):   out[m, n] = sum_k X[m, k] * W[n, k]  (+ R[m, n]),   M = concurrent streams (<= 256).
//
// The step is HBM-bound (each bf16 weight is used for M MACs), so the design goal is to keep
// every SM pulling weight tiles at full rate: the weight matrix is the MMA "A" operand (128 rows of
// W per CTA = two m64 wgmmas), the activations are the "B" operand (wgmma N = M rounded up to 16, 32, 64, 128 or 256),
// both K-major exactly as nn.Linear stores them, 4-stage TMA ring of 128x64 bf16 weight tiles, and split-K across CTAs
// when N/128 alone cannot fill the machine (fp32 partials + finalize kernel).  Every weight tile is read once for all M
// streams: 256 streams cost one pass over the weights, not two.
// Replaces F.linear in CausalSelfAttention / LLaMAMLP / lm_head (models/llama_streaming.py:935-998,
// models/lit_model.py:399-403) and in the depth transformer (modules/transformer.py:155-179, gating.py:12-21).
#include <cuda_bf16.h>

#include <cooperative_groups.h>

#include "common.cuh"
#include "tc_common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {
extern void count_launch();
using namespace tc;

constexpr int SK_BN = 128;      // weight rows per CTA (two m64 wgmmas)
constexpr int SK_BK = 64;       // bf16 elements per 128-byte swizzle row
constexpr int SK_W_BYTES = SK_BN * 128;
constexpr int SK_STAGES = 4;

template <int NB>   // wgmma N: streams rounded up to 16, 32, 64, 128 or 256
struct SkCfg {
  // consumer warpgroups: a 64 x 256 fp32 accumulator is 128 registers per thread, so at NB = 256 each of two warpgroups
  // owns one 64-row half of the weight tile; below, one warpgroup holds both halves
  static constexpr int WG = NB > 128 ? 2 : 1;
  static constexpr int THREADS = 128 * WG + 32;   // + the TMA warp
  static constexpr int MIN_BLOCKS = WG == 1 ? 2 : 1;
  static constexpr int STAGE_BYTES = SK_W_BYTES + ((NB * 128 + 1023) & ~1023);
  static constexpr int SMEM_BYTES = SK_STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

struct SkParams {
  __nv_bfloat16* out;        // [M][N] bf16 (splits == 1)
  float* partial;            // [splits][M][N] fp32 (splits > 1)
  const __nv_bfloat16* R;    // optional residual [M][N]
  int M, N, K;
  int splits, k_iters;       // k_iters = 64-element chunks per split
  int force_partial;         // write fp32 partials even with one split (a fused finalize kernel consumes them)
  int gate_interleaved;      // SiLU gating in the epilogue itself (one split, weight rows interleaved a_0 b_0 a_1 b_1 ...)
  __nv_bfloat16* aux;        // [M][N/2] gated output (gate_interleaved)
};

// Thread roles (160 threads, NB <= 128): warpgroup 0 = consumers (wgmma issue + epilogue), warp 4 = TMA producer.  A
// consumer thread (warp wq, lane = 4 gq + tq) ends with the accumulators of weight rows n0 + 64 h + 16 wq + gq (+ 8),
// streams 8 b + 2 tq (+ 1) for both 64-row halves h.
// NB = 256 (288 threads): warpgroups 0 and 1 are consumers, warpgroup h owning half h only (wq = warp % 4, same row and
// stream mapping), and warp 8 is the TMA producer.  Both warpgroups read the stage's one X tile.
template <int NB>
__global__ void __launch_bounds__(SkCfg<NB>::THREADS, SkCfg<NB>::MIN_BLOCKS)
gemm_skinny_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const SkParams p) {
  constexpr int WG = SkCfg<NB>::WG;
  constexpr int STAGES = SK_STAGES;
  constexpr int STAGE_BYTES = SkCfg<NB>::STAGE_BYTES;
  constexpr int NR = NB / 2;   // accumulator registers per thread of one 64 x NB wgmma
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment (128-byte swizzle atoms) as pointer arithmetic on the __shared__ array (an integer round trip
  // would demote every later access through `smem` to generic LD / ST)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int n0 = blockIdx.x * SK_BN;
  const int split = blockIdx.y;
  const int k_begin = split * p.k_iters;
  int k_count = p.K / SK_BK - k_begin;
  if (k_count > p.k_iters) k_count = p.k_iters;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 4 * WG);   // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 4 * WG) {
    if (elect_one()) {
      tma_prefetch_desc(&tmW);
      tma_prefetch_desc(&tmX);
      for (int kit = 0; kit < k_count; ++kit) {
        const int s = kit % STAGES;
        mbar_wait(&empty[s], ((kit / STAGES) & 1) ^ 1);
        uint8_t* st = smem + s * STAGE_BYTES;
        mbar_arrive_expect_tx(&full[s], SK_W_BYTES + NB * 128);
        tma_load_2d(st, &tmW, &full[s], (k_begin + kit) * SK_BK, n0);
        tma_load_2d(st + SK_W_BYTES, &tmX, &full[s], (k_begin + kit) * SK_BK, 0);
      }
    }
    return;
  }

  // weight rows [0, 64) and [64, 128) of the tile; with two warpgroups, c0 holds the warpgroup's own half and c1 is unused
  float c0[NR], c1[NR];
#pragma unroll
  for (int j = 0; j < NR; ++j) c0[j] = c1[j] = 0.f;
  const uint32_t smem0 = smem_u32(smem);
  const uint32_t half0 = WG == 1 ? 0u : (uint32_t)(warp / 4) * (64 * 128);
  for (int kit = 0; kit < k_count; ++kit) {
    const int s = kit % STAGES;
    mbar_wait(&full[s], (kit / STAGES) & 1);
    const uint32_t st = smem0 + (uint32_t)(s * STAGE_BYTES);
    const uint64_t dw0 = gmma_desc_sw128(st + half0), dw1 = gmma_desc_sw128(st + 64 * 128), dx = gmma_desc_sw128(st + SK_W_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {  // 4 x (K = 16 bf16 = 32 bytes)
      const uint32_t acc_in = (kit > 0 || k > 0) ? 1u : 0u;
      wgmma_bf16_ss<NB>(c0, dw0 + (uint64_t)(2 * k), dx + (uint64_t)(2 * k), acc_in);
      if constexpr (WG == 1) wgmma_bf16_ss<NB>(c1, dw1 + (uint64_t)(2 * k), dx + (uint64_t)(2 * k), acc_in);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_acc(c0);
    if constexpr (WG == 1) fence_acc(c1);
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }

  // epilogue: weight rows n, streams m
  const int gq = lane / 4, tq = lane % 4;
  const int wq = WG == 1 ? warp : warp % 4;
  auto store = [&](const float (&c)[NR], int half) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = n0 + 64 * half + 16 * wq + gq + 8 * e;
      const bool nv = n < p.N;
#pragma unroll
      for (int b = 0; b < NB / 8; ++b) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int m = 8 * b + 2 * tq + u;
          float v = c[4 * b + 2 * e + u];
          if (p.gate_interleaved) {
            // rows 2j / 2j+1 of the interleaved weight are a_j / b_j: lanes 4 apart hold the gate and the value of
            // output column j, so SiLU gating needs one shuffle and no fp32 partials (gating.py:12-21; lit_model.py:399-403)
            const float o = __shfl_xor_sync(0xffffffffu, v, 4);
            if (!(gq & 1) && nv && m < p.M) {
              const int I = p.N / 2;
              const float a = __bfloat162float(__float2bfloat16(v)), bb = __bfloat162float(__float2bfloat16(o));
              const float sl = __bfloat162float(__float2bfloat16(a / (1.0f + expf(-a))));
              p.aux[(long long)m * I + (n >> 1)] = __float2bfloat16(sl * bb);
            }
          } else if (nv && m < p.M) {
            if (p.splits > 1 || p.force_partial) {
              p.partial[((long long)split * p.M + m) * p.N + n] = v;
            } else {
              if (p.R) v += __bfloat162float(p.R[(long long)m * p.N + n]);
              p.out[(long long)m * p.N + n] = __float2bfloat16(v);
            }
          }
        }
      }
    }
  };
  store(c0, WG == 1 ? 0 : warp / 4);
  if constexpr (WG == 1) store(c1, 1);
}

// plain finalize: out = bf16(sum_s partial[s] + R), 4 elements per thread (N % 4 == 0)
__global__ void skinny_finalize_kernel(const float* __restrict__ partial, const __nv_bfloat16* __restrict__ R,
                                       __nv_bfloat16* __restrict__ out, long long MN, int splits) {
  const long long n4 = MN / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 v = *reinterpret_cast<const float4*>(partial + 4 * i);
    for (int s = 1; s < splits; ++s) {
      const float4 t = *reinterpret_cast<const float4*>(partial + (long long)s * MN + 4 * i);
      v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
    }
    if (R) {
      const __nv_bfloat162* r2 = reinterpret_cast<const __nv_bfloat162*>(R + 4 * i);
      const float2 a = __bfloat1622float2(r2[0]), b = __bfloat1622float2(r2[1]);
      v.x += a.x; v.y += a.y; v.z += b.x; v.w += b.y;
    }
    __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(out + 4 * i);
    o2[0] = __floats2bfloat162_rn(v.x, v.y);
    o2[1] = __floats2bfloat162_rn(v.z, v.w);
  }
}

// finalize + residual + RMSNorm of the result in one pass over the row:
//   out[m] = bf16(sum_s partial[s][m] + R[m]);  aux[m] = rmsnorm(out[m]) * w   (the NEXT op's pre-norm)
// Replaces three kernels (finalize, residual add, RMSNorm) between a projection and the following GEMM.
// A cluster of FIN_CL CTAs shares one row (M = 64 rows alone would leave most SMs idle): each CTA reduces its column
// slice, the slice sums of squares are exchanged through distributed shared memory and added in rank order, so the
// result does not depend on timing.
constexpr int FIN_CL = 4;
__global__ void __cluster_dims__(FIN_CL, 1, 1)
skinny_finalize_norm_kernel(const float* __restrict__ partial, const __nv_bfloat16* __restrict__ R,
                            __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ w,
                            __nv_bfloat16* __restrict__ aux, int M, int N, int splits, float eps, int kyutai) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ float red[32];
  __shared__ float slice_ss;
  const int m = blockIdx.x / FIN_CL, slice = (int)cluster.block_rank();
  const int n_lo = slice * (N / FIN_CL), n_hi = n_lo + N / FIN_CL;
  const long long MN = (long long)M * N;
  float ss = 0.f;
  for (int n = n_lo + threadIdx.x * 4; n < n_hi; n += blockDim.x * 4) {
    const long long i = (long long)m * N + n;
    float4 v = *reinterpret_cast<const float4*>(partial + i);
    for (int s = 1; s < splits; ++s) {
      const float4 t = *reinterpret_cast<const float4*>(partial + (long long)s * MN + i);
      v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
    }
    if (R) {
      const __nv_bfloat162* r2 = reinterpret_cast<const __nv_bfloat162*>(R + i);
      const float2 a = __bfloat1622float2(r2[0]), b = __bfloat1622float2(r2[1]);
      v.x += a.x; v.y += a.y; v.z += b.x; v.w += b.y;
    }
    const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(out + i);
    o2[0] = lo; o2[1] = hi;
    const float2 fa = __bfloat1622float2(lo), fb = __bfloat1622float2(hi);  // the norm sees the stored bf16 values
    ss = fmaf(fa.x, fa.x, ss); ss = fmaf(fa.y, fa.y, ss); ss = fmaf(fb.x, fb.x, ss); ss = fmaf(fb.y, fb.y, ss);
  }
  ss = warp_sum(ss);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < blockDim.x / 32 ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) slice_ss = t;
  }
  cluster.sync();
  float tot = 0.f;
#pragma unroll
  for (int r = 0; r < FIN_CL; ++r) tot += *cluster.map_shared_rank(&slice_ss, r);
  cluster.sync();   // nobody leaves (and frees its shared memory) while a peer may still be reading it
  const float mean = tot / (float)N;
  const float r = kyutai ? rsqrtf(eps + mean) : rsqrtf(mean + eps);
  for (int n = n_lo + threadIdx.x * 4; n < n_hi; n += blockDim.x * 4) {
    const long long i = (long long)m * N + n;
    const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(out + i);
    const __nv_bfloat162* w2 = reinterpret_cast<const __nv_bfloat162*>(w + n);
    const float2 xa = __bfloat1622float2(x2[0]), xb = __bfloat1622float2(x2[1]);
    const float2 wa = __bfloat1622float2(w2[0]), wb = __bfloat1622float2(w2[1]);
    float4 o;
    if (kyutai) { o.x = xa.x * (wa.x * r); o.y = xa.y * (wa.y * r); o.z = xb.x * (wb.x * r); o.w = xb.y * (wb.y * r); }
    else        { o.x = (xa.x * r) * wa.x; o.y = (xa.y * r) * wa.y; o.z = (xb.x * r) * wb.x; o.w = (xb.y * r) * wb.y; }
    __nv_bfloat162* a2 = reinterpret_cast<__nv_bfloat162*>(aux + i);
    a2[0] = __floats2bfloat162_rn(o.x, o.y);
    a2[1] = __floats2bfloat162_rn(o.z, o.w);
  }
}

// finalize + SiLU gating: aux[m][c] = bf16(silu(bf16(a)) ) * bf16(b) with a = cols [0,I), b = cols [I,2I) of the GEMM result
__global__ void skinny_finalize_silu_kernel(const float* __restrict__ partial, __nv_bfloat16* __restrict__ aux, int M, int N,
                                            int splits) {
  const int I = N / 2;
  const long long MN = (long long)M * N, total = (long long)M * I;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / I, c = i % I;
    float a = 0.f, b = 0.f;
    for (int s = 0; s < splits; ++s) {
      a += partial[(long long)s * MN + m * N + c];
      b += partial[(long long)s * MN + m * N + I + c];
    }
    a = __bfloat162float(__float2bfloat16(a));
    b = __bfloat162float(__float2bfloat16(b));
    const float sl = __bfloat162float(__float2bfloat16(a / (1.0f + expf(-a))));
    aux[i] = __float2bfloat16(sl * b);
  }
}

typedef CUresult (*EncodeTiledFn2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn2 get_encode_fn2() {
  static EncodeTiledFn2 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && p) fn = (EncodeTiledFn2)p;
  }
  return fn;
}

typedef void (*SkinnyKernel)(const CUtensorMap, const CUtensorMap, const SkParams);
static SkinnyKernel skinny_kernel(int nb) {
  switch (nb) {
    case 16: return gemm_skinny_kernel<16>;
    case 32: return gemm_skinny_kernel<32>;
    case 64: return gemm_skinny_kernel<64>;
    case 128: return gemm_skinny_kernel<128>;
    default: return gemm_skinny_kernel<256>;
  }
}
static int skinny_smem(int nb) {
  switch (nb) {
    case 16: return SkCfg<16>::SMEM_BYTES;
    case 32: return SkCfg<32>::SMEM_BYTES;
    case 64: return SkCfg<64>::SMEM_BYTES;
    case 128: return SkCfg<128>::SMEM_BYTES;
    default: return SkCfg<256>::SMEM_BYTES;
  }
}
static int skinny_threads(int nb) { return nb > 128 ? SkCfg<256>::THREADS : SkCfg<128>::THREADS; }
// one-time opt-in to the instantiation's dynamic shared memory (per device, like smem_optin)
static void skinny_optin(int nb) {
  static unsigned long long done[5] = {0, 0, 0, 0, 0};
  const int idx = nb == 16 ? 0 : nb == 32 ? 1 : nb == 64 ? 2 : nb == 128 ? 3 : 4;
  smem_optin(skinny_kernel(nb), skinny_smem(nb), done[idx]);
}
}  // namespace rstnet
using namespace rstnet;

struct rstnet_skinny_plan {
  CUtensorMap tmW, tmX;
  SkParams p;
  dim3 grid;
  size_t smem;
  int nb;        // wgmma N (streams rounded up)
  int fin_mode;  // 0 plain, 1 finalize + residual + RMSNorm -> aux, 2 finalize + SiLU gating -> aux, 3 gating in the epilogue
  const __nv_bfloat16* norm_w;
  __nv_bfloat16* aux;
  float eps;
  int kyutai;
};

extern "C" int rstnet_skinny_gemm_create_fused(const void* X, const void* W, const void* R, void* out, float* partial_ws,
                                               int32_t M, int32_t N, int32_t K, int32_t max_splits, int32_t fin_mode,
                                               const void* norm_w, void* aux_out, float eps, int32_t kyutai,
                                               rstnet_skinny_plan** outp);

extern "C" int rstnet_skinny_gemm_create(const void* X, const void* W, const void* R, void* out, float* partial_ws,
                                         int32_t M, int32_t N, int32_t K, int32_t max_splits, rstnet_skinny_plan** outp) {
  return rstnet_skinny_gemm_create_fused(X, W, R, out, partial_ws, M, N, K, max_splits, 0, nullptr, nullptr, 0.f, 0, outp);
}

extern "C" int rstnet_skinny_gemm_create_fused(const void* X, const void* W, const void* R, void* out, float* partial_ws,
                                               int32_t M, int32_t N, int32_t K, int32_t max_splits, int32_t fin_mode,
                                               const void* norm_w, void* aux_out, float eps, int32_t kyutai,
                                               rstnet_skinny_plan** outp) {
  RSTNET_REQUIRE(X && W && outp && (out || fin_mode >= 2), "skinny_gemm_create: null pointer");
  RSTNET_REQUIRE(fin_mode >= 0 && fin_mode <= 3, "skinny_gemm_create: bad fin_mode");
  if (fin_mode == 3) {   // SiLU gating on interleaved weight rows, finished in the GEMM epilogue: one K slice, no workspace
    RSTNET_REQUIRE(aux_out && N % 2 == 0, "skinny_gemm_create: interleaved SiLU gating needs an aux output and an even N (N=%d)", N);
    partial_ws = nullptr;
    max_splits = 1;
  }
  RSTNET_REQUIRE(fin_mode != 1 || N % (4 * FIN_CL) == 0, "skinny_gemm_create: fused RMSNorm needs N %% 16 == 0 (N=%d)", N);
  RSTNET_REQUIRE(fin_mode == 0 || fin_mode == 3 || (partial_ws && aux_out && N % 4 == 0 && (fin_mode == 2 || norm_w)),
                 "skinny_gemm_create: fused finalize needs a workspace, an aux output and N %% 4 == 0");
  RSTNET_REQUIRE(M >= 1 && M <= 256 && N >= 1 && K >= SK_BK && K % SK_BK == 0, "skinny_gemm_create: need 1<=M<=256, K %% 64 == 0 (M=%d N=%d K=%d)", M, N, K);
  RSTNET_REQUIRE((uintptr_t)X % 16 == 0 && (uintptr_t)W % 16 == 0, "skinny_gemm_create: X and W must be 16-byte aligned");
  EncodeTiledFn2 enc = get_encode_fn2();
  RSTNET_REQUIRE(enc != nullptr, "skinny_gemm_create: cuTensorMapEncodeTiled unavailable");
  rstnet_skinny_plan* pl = new rstnet_skinny_plan();
  const int NB = M <= 16 ? 16 : M <= 32 ? 32 : M <= 64 ? 64 : M <= 128 ? 128 : 256;
  const int n_tiles = ceil_div(N, SK_BN);
  const int kchunks = K / SK_BK;
  int splits = 1;
  RSTNET_REQUIRE(!(partial_ws && max_splits > 1) || N % 4 == 0, "skinny_gemm_create: split-K needs N %% 4 == 0");
  if (partial_ws && max_splits > 1) {
    // Enough CTAs to keep ~1.5 per SM streaming, no more: every split adds an fp32 partial round trip.
    const int cand[6] = {1, 2, 3, 4, 6, 8};
    const float want = 1.5f * (float)sm_count() / (float)n_tiles;
    float best = 1e30f;
    for (int c : cand) {
      if (c > max_splits || (c > 1 && kchunks / c < 8)) continue;
      // M > 128 runs one CTA per SM, and a split count whose CTAs need a second wave (n_tiles * c > SMs) waits for it:
      // at the Llama-3.2-3B widths with M = 256 on an H100 the 1.5-per-SM choice took 1.8-1.9x the time of the best
      // split count (QKV, N 5120 K 3072: 6 splits 0.117 ms, 3 splits 0.061 ms).  The largest one-wave count left (the
      // closest to `want`) was the fastest measured for 7 of the 8 split-K shapes of that model and within 15 % for the
      // other one (attention proj: 4 splits 0.058 ms, 3 splits 0.051 ms).
      if (NB == 256 && c > 1 && c * n_tiles > sm_count()) continue;
      const float r = (float)c > want ? (float)c / want : want / (float)c;
      if (r < best) { best = r; splits = c; }
    }
    // every split must own at least one K chunk (a CTA without work would never signal its accumulator)
    while (splits > 1 && (splits - 1) * ceil_div(kchunks, splits) >= kchunks) --splits;
  }
  {
    cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)N};
    cuuint64_t gstr[1] = {(cuuint64_t)K * 2};
    cuuint32_t box[2] = {SK_BK, SK_BN};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&pl->tmW, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)W, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    cuuint64_t gdx[2] = {(cuuint64_t)K, (cuuint64_t)M};
    cuuint32_t bx[2] = {SK_BK, (cuuint32_t)NB};
    if (r == CUDA_SUCCESS)
      r = enc(&pl->tmX, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)X, gdx, gstr, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      delete pl;
      set_error("skinny_gemm_create: cuTensorMapEncodeTiled failed with %d", (int)r);
      return 3;
    }
  }
  SkParams& p = pl->p;
  p.out = (__nv_bfloat16*)out; p.partial = partial_ws; p.R = (const __nv_bfloat16*)R;
  p.M = M; p.N = N; p.K = K; p.splits = splits;
  p.gate_interleaved = fin_mode == 3; p.aux = (__nv_bfloat16*)aux_out;
  pl->nb = NB;
  pl->fin_mode = fin_mode; pl->norm_w = (const __nv_bfloat16*)norm_w; pl->aux = (__nv_bfloat16*)aux_out; pl->eps = eps; pl->kyutai = kyutai;
  // a fused finalize always reads fp32 partials, so the main kernel takes the split path even with one split
  p.force_partial = fin_mode == 1 || fin_mode == 2;
  p.k_iters = ceil_div(kchunks, splits);
  pl->grid = dim3((unsigned)n_tiles, (unsigned)splits);
  // 4 stages (<= 98 KB with M <= 64): two CTAs fit per SM, so a GEMM whose tile count is not a multiple of the SM count
  // still keeps every SM streaming (bandwidth-bound CTAs progress at equal rates) and prologues overlap main loops.
  // M = 65..128 (130 KB) and 129..256 (194 KB) run one CTA per SM.
  pl->smem = (size_t)skinny_smem(NB);
  *outp = pl;
  return 0;
}

extern "C" int rstnet_skinny_gemm_run(const rstnet_skinny_plan* pl, rstnet_stream_t stream) {
  RSTNET_REQUIRE(pl != nullptr, "skinny_gemm_run: null plan");
  skinny_optin(pl->nb);
  cudaStream_t st = (cudaStream_t)stream;
  skinny_kernel(pl->nb)<<<pl->grid, dim3(skinny_threads(pl->nb)), pl->smem, st>>>(pl->tmW, pl->tmX, pl->p);
  count_launch();
  if (int e = check_launch("gemm_skinny")) return e;
  const long long MN = (long long)pl->p.M * pl->p.N;
  if (pl->fin_mode == 1) {
    skinny_finalize_norm_kernel<<<dim3(pl->p.M * FIN_CL), dim3(256), 0, st>>>((const float*)pl->p.partial, pl->p.R, pl->p.out, pl->norm_w,
                                                                              pl->aux, pl->p.M, pl->p.N, pl->p.splits, pl->eps, pl->kyutai);
    count_launch();
    return check_launch("skinny_finalize_norm");
  }
  if (pl->fin_mode == 2) {
    int g = ceil_div(MN / 2, 256);
    if (g > sm_count() * 8) g = sm_count() * 8;
    skinny_finalize_silu_kernel<<<dim3(g), dim3(256), 0, st>>>((const float*)pl->p.partial, pl->aux, pl->p.M, pl->p.N, pl->p.splits);
    count_launch();
    return check_launch("skinny_finalize_silu");
  }
  if (pl->p.splits > 1) {
    int g = ceil_div(MN / 4, 256);
    if (g > sm_count() * 4) g = sm_count() * 4;
    skinny_finalize_kernel<<<dim3(g), dim3(256), 0, st>>>((const float*)pl->p.partial, pl->p.R, pl->p.out, MN, pl->p.splits);
    count_launch();
    return check_launch("skinny_finalize");
  }
  return 0;
}

extern "C" void rstnet_skinny_gemm_destroy(rstnet_skinny_plan* pl) {
  delete pl;
}
extern "C" int64_t rstnet_skinny_gemm_workspace(int32_t M, int32_t N, int32_t max_splits) {
  return (int64_t)max_splits * M * N * (int64_t)sizeof(float);
}
