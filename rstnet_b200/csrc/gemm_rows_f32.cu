// Strided-row fp32 GEMM on the CUDA cores: every causal conv / transposed conv / linear of the
// Mimi codec (see include/rstnet_b200.h).  fp32 FFMA is deliberate for the encoder side: RVQ
// indices must match the reference bit-for-bit, which rules out TF32/BF16 inputs (SURVEY.md H1).
//
// Tiling: BM x BN output tile per CTA, BK = 16, 3-stage cp.async pipeline, TM x TN register
// micro-tile per thread.  A rows are fetched straight from the overlapping conv windows
// (row base = b*a_batch_stride + t*a_row_stride), so no im2col buffer ever exists in HBM.
#include "common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {

extern void count_launch();

template <int BM_, int BN_, int TM_, int TN_>
struct TileCfg {
  static constexpr int BM = BM_, BN = BN_, TM = TM_, TN = TN_;
  static constexpr int BK = 16;
  static constexpr int NTX = BN / TN, NTY = BM / TM, NT = NTX * NTY;
  static constexpr int AS = BK + 4;  // padded A row stride in smem (floats), keeps 16B alignment
  static constexpr int STAGES = 3;
  static constexpr int A_STAGE = BM * AS, B_STAGE = BK * BN;
  static constexpr int SMEM_BYTES = STAGES * (A_STAGE + B_STAGE) * 4;
  static constexpr int A_CHUNKS = BM * (BK / 4);
  static constexpr int B_CHUNKS = BK * (BN / 4);
  static constexpr int A_PER_T = (A_CHUNKS + NT - 1) / NT;
  static constexpr int B_PER_T = (B_CHUNKS + NT - 1) / NT;
  static_assert(TN % 4 == 0, "TN must be a multiple of 4");
};

template <class Cfg>
__global__ void __launch_bounds__(Cfg::NT) gemm_rows_kernel(const rstnet_gemm_rows_args p) {
  constexpr int BM = Cfg::BM, BN = Cfg::BN, TM = Cfg::TM, TN = Cfg::TN, BK = Cfg::BK;
  constexpr int NTX = Cfg::NTX, NTY = Cfg::NTY, NT = Cfg::NT, AS = Cfg::AS, STAGES = Cfg::STAGES;
  extern __shared__ __align__(16) float smem[];
  float* As = smem;
  float* Bs = smem + STAGES * Cfg::A_STAGE;

  const int tid = threadIdx.x;
  const int tx = tid % NTX, ty = tid / NTX;
  const long long M = (long long)p.batch * p.rows;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int K = p.K, N = p.N;
  const int kc = p.taps > 1 ? p.K / p.taps : p.K;
  const long long tap_stride = p.taps > 1 ? p.tap_stride : 0;

  // ---- per-thread copy assignments (fixed across k tiles)
  const float* a_src[Cfg::A_PER_T];
  int a_dst[Cfg::A_PER_T];
  int a_q[Cfg::A_PER_T];
#pragma unroll
  for (int i = 0; i < Cfg::A_PER_T; ++i) {
    int c = tid + i * NT;
    int row = c / (BK / 4), q = c % (BK / 4);
    if (c >= Cfg::A_CHUNKS) { row = 0; q = 0; }
    long long m = m0 + row;
    if (m >= M) m = M - 1;
    long long b = m / p.rows, t = m % p.rows;
    a_src[i] = p.A + b * p.a_batch_stride + t * p.a_row_stride;
    a_dst[i] = row * AS + 4 * q;
    a_q[i] = q;
  }
  int b_src[Cfg::B_PER_T];
  int b_dst[Cfg::B_PER_T];
  int b_k[Cfg::B_PER_T];
  bool b_ok[Cfg::B_PER_T];
#pragma unroll
  for (int i = 0; i < Cfg::B_PER_T; ++i) {
    int c = tid + i * NT;
    int k = c / (BN / 4), nq = c % (BN / 4);
    if (c >= Cfg::B_CHUNKS) { k = 0; nq = 0; }
    int n = n0 + 4 * nq;
    b_ok[i] = (n < N) && (c < Cfg::B_CHUNKS);
    b_src[i] = k * N + (n < N ? n : 0);
    b_dst[i] = k * BN + 4 * nq;
    b_k[i] = k;
  }

  auto load_stage = [&](int kt, int stage) {
    float* as = As + stage * Cfg::A_STAGE;
    float* bs = Bs + stage * Cfg::B_STAGE;
    const int k0 = kt * BK;
#pragma unroll
    for (int i = 0; i < Cfg::A_PER_T; ++i) {
      if (tid + i * NT < Cfg::A_CHUNKS) {
        int kk = k0 + 4 * a_q[i];
        bool ok = kk < K;
        // K index -> (tap, channel): taps are tap_stride elements apart (time-major layout); a 4-float
        // chunk never straddles taps because kc % 4 == 0
        const int tap = kk / kc, c = kk - tap * kc;
        cp_async16(as + a_dst[i], ok ? (const void*)(a_src[i] + (long long)tap * tap_stride + c) : (const void*)p.A, ok ? 16 : 0);
      }
    }
#pragma unroll
    for (int i = 0; i < Cfg::B_PER_T; ++i) {
      if (tid + i * NT < Cfg::B_CHUNKS) {
        bool ok = b_ok[i] && (k0 + b_k[i] < K);
        cp_async16(bs + b_dst[i], ok ? (const void*)(p.Wt + (long long)k0 * N + b_src[i]) : (const void*)p.Wt,
                   ok ? 16 : 0);
      }
    }
  };

  const int KT = (K + BK - 1) / BK;
#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < KT) load_stage(s, s);
    cp_async_commit();
  }

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  const int pre_act = p.pre_act;
  for (int kt = 0; kt < KT; ++kt) {
    const int stage = kt % STAGES;
    cp_async_wait<STAGES - 2>();
    if (pre_act != ACT_NONE) {
      // the issuing thread sees its own completed cp.async data: activate it in place
      float* as = As + stage * Cfg::A_STAGE;
#pragma unroll
      for (int i = 0; i < Cfg::A_PER_T; ++i) {
        if (tid + i * NT < Cfg::A_CHUNKS) {
          float4 v = *reinterpret_cast<float4*>(as + a_dst[i]);
          v.x = apply_act(v.x, pre_act); v.y = apply_act(v.y, pre_act);
          v.z = apply_act(v.z, pre_act); v.w = apply_act(v.w, pre_act);
          *reinterpret_cast<float4*>(as + a_dst[i]) = v;
        }
      }
    }
    __syncthreads();
    {
      const int nk = kt + STAGES - 1;
      if (nk < KT) load_stage(nk, nk % STAGES);
      cp_async_commit();
    }
    const float* as = As + stage * Cfg::A_STAGE;
    const float* bs = Bs + stage * Cfg::B_STAGE;
#pragma unroll
    for (int kk = 0; kk < BK; kk += 4) {
      float4 a[TM];
#pragma unroll
      for (int i = 0; i < TM; ++i) a[i] = *reinterpret_cast<const float4*>(as + (ty + i * NTY) * AS + kk);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        float4 b[TN / 4];
#pragma unroll
        for (int j = 0; j < TN / 4; ++j)
          b[j] = *reinterpret_cast<const float4*>(bs + (kk + c) * BN + tx * 4 + j * (NTX * 4));
#pragma unroll
        for (int i = 0; i < TM; ++i) {
          const float av = c == 0 ? a[i].x : (c == 1 ? a[i].y : (c == 2 ? a[i].z : a[i].w));
#pragma unroll
          for (int j = 0; j < TN / 4; ++j) {
            acc[i][4 * j + 0] = fmaf(av, b[j].x, acc[i][4 * j + 0]);
            acc[i][4 * j + 1] = fmaf(av, b[j].y, acc[i][4 * j + 1]);
            acc[i][4 * j + 2] = fmaf(av, b[j].z, acc[i][4 * j + 2]);
            acc[i][4 * j + 3] = fmaf(av, b[j].w, acc[i][4 * j + 3]);
          }
        }
      }
    }
  }
  cp_async_wait<0>();

  // ---- epilogue: bias, LayerScale, residual, activation; float4 stores along N
  const int post_act = p.post_act;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const long long m = m0 + ty + i * NTY;
    if (m >= M) continue;
    const long long b = m / p.rows, t = m % p.rows;
    float* crow = p.C + b * p.c_batch_stride + t * p.c_row_stride;
    const float* rrow = p.R ? p.R + b * p.r_batch_stride + t * p.r_row_stride : nullptr;
#pragma unroll
    for (int j = 0; j < TN / 4; ++j) {
      const int n = n0 + tx * 4 + j * (NTX * 4);
      if (n >= N) continue;
      float4 v = make_float4(acc[i][4 * j], acc[i][4 * j + 1], acc[i][4 * j + 2], acc[i][4 * j + 3]);
      if (p.bias) {
        const float4 bb = *reinterpret_cast<const float4*>(p.bias + n);
        v.x += bb.x; v.y += bb.y; v.z += bb.z; v.w += bb.w;
      }
      if (p.scale) {
        const float4 ss = *reinterpret_cast<const float4*>(p.scale + n);
        v.x *= ss.x; v.y *= ss.y; v.z *= ss.z; v.w *= ss.w;
      }
      if (rrow) {
        const float4 rr = *reinterpret_cast<const float4*>(rrow + n);
        v.x += rr.x; v.y += rr.y; v.z += rr.z; v.w += rr.w;
      }
      if (post_act != ACT_NONE) {
        v.x = apply_act(v.x, post_act); v.y = apply_act(v.y, post_act);
        v.z = apply_act(v.z, post_act); v.w = apply_act(v.w, post_act);
      }
      *reinterpret_cast<float4*>(crow + n) = v;
    }
  }
}

template <class Cfg>
static int launch_cfg(const rstnet_gemm_rows_args& a, cudaStream_t st) {
  static unsigned long long attr_done = 0;  // per instantiation and per device; benign if raced
  smem_optin(gemm_rows_kernel<Cfg>, Cfg::SMEM_BYTES, attr_done);
  const long long M = (long long)a.batch * a.rows;
  dim3 grid((unsigned)ceil_div(M, Cfg::BM), (unsigned)ceil_div(a.N, Cfg::BN));
  gemm_rows_kernel<Cfg><<<grid, Cfg::NT, Cfg::SMEM_BYTES, st>>>(a);
  count_launch();
  return check_launch("gemm_rows_f32");
}

}  // namespace rstnet

using namespace rstnet;

extern "C" int rstnet_gemm_rows_f32(const rstnet_gemm_rows_args* args, rstnet_stream_t stream) {
  RSTNET_REQUIRE(args != nullptr, "gemm_rows: null args");
  const rstnet_gemm_rows_args& a = *args;
  RSTNET_REQUIRE(a.A && a.Wt && a.C, "gemm_rows: null pointer");
  RSTNET_REQUIRE(a.batch > 0 && a.rows > 0 && a.N > 0 && a.K > 0, "gemm_rows: empty problem (batch=%d rows=%d N=%d K=%d)",
                 a.batch, a.rows, a.N, a.K);
  RSTNET_REQUIRE(a.K % 4 == 0 && a.N % 4 == 0, "gemm_rows: K (%d) and N (%d) must be multiples of 4", a.K, a.N);
  RSTNET_REQUIRE(a.taps <= 1 || (a.K % a.taps == 0 && (a.K / a.taps) % 4 == 0 && a.tap_stride % 4 == 0),
                 "gemm_rows: with taps, K/taps and tap_stride must be multiples of 4");
  RSTNET_REQUIRE(a.a_batch_stride % 4 == 0 && a.a_row_stride % 4 == 0 && a.c_batch_stride % 4 == 0 &&
                     a.c_row_stride % 4 == 0 && a.r_batch_stride % 4 == 0 && a.r_row_stride % 4 == 0,
                 "gemm_rows: strides must be multiples of 4 elements (16-byte rows)");
  RSTNET_REQUIRE(((uintptr_t)a.A % 16 == 0) && ((uintptr_t)a.Wt % 16 == 0) && ((uintptr_t)a.C % 16 == 0) &&
                     ((uintptr_t)a.R % 16 == 0) && ((uintptr_t)a.bias % 16 == 0) && ((uintptr_t)a.scale % 16 == 0),
                 "gemm_rows: pointers must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const long long M = (long long)a.batch * a.rows;
  const int N = a.N;
  // Tile choice: widest tile that still gives >= 2 CTAs per SM; narrow N gets narrow BN.
  auto ctas = [&](int bm, int bn) { return (long long)ceil_div(M, bm) * ceil_div(N, bn); };
  const long long want = 2 * sm_count();
  if (N <= 32) {
    if (ctas(128, 32) >= want) return launch_cfg<TileCfg<128, 32, 4, 4>>(a, st);
    return launch_cfg<TileCfg<32, 32, 2, 4>>(a, st);
  }
  if (N <= 64) {
    if (ctas(128, 64) >= want) return launch_cfg<TileCfg<128, 64, 8, 4>>(a, st);
    if (ctas(64, 64) >= want) return launch_cfg<TileCfg<64, 64, 4, 4>>(a, st);
    return launch_cfg<TileCfg<32, 64, 2, 4>>(a, st);
  }
  if (ctas(128, 128) >= want) return launch_cfg<TileCfg<128, 128, 8, 8>>(a, st);
  if (ctas(128, 64) >= want) return launch_cfg<TileCfg<128, 64, 8, 4>>(a, st);
  if (ctas(64, 64) >= want) return launch_cfg<TileCfg<64, 64, 4, 4>>(a, st);
  if (ctas(32, 64) >= want) return launch_cfg<TileCfg<32, 64, 2, 4>>(a, st);
  return launch_cfg<TileCfg<32, 32, 2, 4>>(a, st);
}
