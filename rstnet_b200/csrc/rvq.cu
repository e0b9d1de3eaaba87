// Split residual vector quantizer: nearest-centroid search (encode) and centroid gather (decode).
// Reference: SplitResidualVectorQuantizer.encode/decode (quantization/vq.py:305-323),
// ResidualVectorQuantization.encode (quantization/core_vq.py:365-376), EuclideanCodebook._quantize
// (core_vq.py:179-185: torch.cdist(p=2) + argmin, first minimum wins).
//
// One launch per residual level.  grid = (frames/32, bins/128): every CTA first rebuilds the
// residual of its 32 frames from the previous level's winners (reducing that level's per-chunk
// partial minima), then scores them against a 128-centroid chunk with an fp32 FFMA GEMM
// (K = dim, centroids streamed k-major through a 3-stage cp.async pipeline), and writes one
// (distance, index) partial per frame.  Splitting bins across CTAs is what keeps every SM busy in
// the streaming regime (N = concurrent streams, e.g. 256 frames per step); codebooks (16 MiB)
// stay L2-resident.  Distances use torch.cdist's matmul form so near-ties resolve the same way:
// d = sqrt(max(|x|^2 + |e|^2 - 2 x.e, 0)).
#include "common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {
extern void count_launch();

constexpr int RQ_BM = 32;    // frames per CTA
constexpr int RQ_BN = 128;   // centroids per CTA
constexpr int RQ_BK = 16;
constexpr int RQ_NT = 256;   // 8 warps; warp w owns rows {w, w+8, w+16, w+24}, lane owns 4 centroids
constexpr int RQ_STAGES = 3;

struct RvqLevelParams {
  const float* x_first;     // level is first of its group: residual = x_first[n*ldx + 0..dim)
  long long ldx;
  const float* r_prev;      // else: residual = r_prev[n] - e_prev[code_prev[n]]
  float* r_cur;             // written by blockIdx.y == 0 (next level reads it)
  const float* e_prev;      // [bins][dim] centroids of the previous level
  const float* pval_prev;   // [N][nch] partial minima of the previous level
  const int* pidx_prev;
  long long* codes;         // [B][n_q][T]
  int prev_level;           // code slot written from the previous level's winners
  const float* et;          // [dim][bins] this level's centroids, k-major
  const float* enorm;       // [bins]
  float* pval;              // [N][nch] out
  int* pidx;
  long long N;
  int T, n_q, dim, bins, nch;
  int time_major;  // frame n = t*B + b instead of b*T + t
};

__device__ __forceinline__ void argmin_combine(float& v, int& i, float ov, int oi) {
  if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
}

__global__ void __launch_bounds__(RQ_NT) rvq_level_kernel(const RvqLevelParams p) {
  extern __shared__ __align__(16) float smem[];
  const int dim = p.dim, RS = dim + 4;
  float* rs = smem;                               // [RQ_BM][dim+4]  holds -2 * residual
  float* xnorm = rs + RQ_BM * RS;                 // [RQ_BM]
  int* code_s = reinterpret_cast<int*>(xnorm + RQ_BM);  // [RQ_BM]
  float* Bs = xnorm + 2 * RQ_BM;                  // [STAGES][BK][BN]
  const int tid = threadIdx.x, lane = tid % 32, warp = tid / 32;
  const long long n0 = (long long)blockIdx.x * RQ_BM;
  const int c0 = blockIdx.y * RQ_BN;

  // ---- B-tile copy assignment: BK*BN/4 = 512 float4 chunks per stage, 2 per thread
  auto load_b = [&](int kt, int stage) {
    float* bs = Bs + stage * RQ_BK * RQ_BN;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int c = tid + i * RQ_NT;
      const int k = c / (RQ_BN / 4), nq = c % (RQ_BN / 4);
      const int kg = kt * RQ_BK + k;
      const bool ok = kg < dim;
      cp_async16(bs + k * RQ_BN + 4 * nq, ok ? (const void*)(p.et + (long long)kg * p.bins + c0 + 4 * nq) : (const void*)p.et,
                 ok ? 16 : 0);
    }
  };
  const int KT = (dim + RQ_BK - 1) / RQ_BK;
#pragma unroll
  for (int s = 0; s < RQ_STAGES - 1; ++s) {
    if (s < KT) load_b(s, s);
    cp_async_commit();
  }

  // ---- previous level's winner per frame (first-minimum across chunks, chunks are index-ordered)
  if (p.x_first == nullptr) {
    for (int r = warp; r < RQ_BM; r += RQ_NT / 32) {
      const long long n = n0 + r;
      float v = INFINITY;
      int idx = 0x7fffffff;
      if (n < p.N) {
        for (int c = lane; c < p.nch; c += 32) argmin_combine(v, idx, p.pval_prev[n * p.nch + c], p.pidx_prev[n * p.nch + c]);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        argmin_combine(v, idx, ov, oi);
      }
      if (lane == 0) {
        // every d is a number, so the argmin always takes a candidate and idx is in [0, bins); the check keeps the
        // centroid gather below in bounds should that ever stop holding (the code written out still shows it)
        code_s[r] = (n < p.N && idx >= 0 && idx < p.bins) ? idx : 0;
        if (blockIdx.y == 0 && n < p.N) {
          const long long nb = p.N / p.T;
          const long long b = p.time_major ? n % nb : n / p.T, t = p.time_major ? n / nb : n % p.T;
          p.codes[(b * p.n_q + p.prev_level) * p.T + t] = idx;
        }
      }
    }
    __syncthreads();
  }

  // ---- residual tile: r = x (first level of the group) or r_prev - e_prev[code] (core_vq.py:372-373)
  const int d4n = dim / 4;
  for (int i = tid; i < RQ_BM * d4n; i += RQ_NT) {
    const int r = i / d4n, d4 = i % d4n;
    const long long n = n0 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n < p.N) {
      if (p.x_first) {
        v = *reinterpret_cast<const float4*>(p.x_first + n * p.ldx + 4 * d4);
      } else {
        const float4 a = *reinterpret_cast<const float4*>(p.r_prev + n * dim + 4 * d4);
        const float4 e = *reinterpret_cast<const float4*>(p.e_prev + (long long)code_s[r] * dim + 4 * d4);
        v = make_float4(a.x - e.x, a.y - e.y, a.z - e.z, a.w - e.w);
      }
      if (blockIdx.y == 0) *reinterpret_cast<float4*>(p.r_cur + n * dim + 4 * d4) = v;
    }
    // -2*x is exact in binary floating point, so fma(-2x, e, acc) == torch's x1_ = cat([-2*x, ...]) matmul terms
    *reinterpret_cast<float4*>(rs + r * RS + 4 * d4) = make_float4(-2.f * v.x, -2.f * v.y, -2.f * v.z, -2.f * v.w);
  }
  __syncthreads();
  for (int r = warp; r < RQ_BM; r += RQ_NT / 32) {
    float s = 0.f;
    for (int d = lane; d < dim; d += 32) { const float h = -0.5f * rs[r * RS + d]; s = fmaf(h, h, s); }
    s = warp_sum(s);
    if (lane == 0) xnorm[r] = s;
  }
  // (xnorm is consumed after the k loop, which contains __syncthreads)

  // ---- scores: acc[i][e] = sum_k (-2 r[row_i][k]) * et[k][c0 + 4*lane + e]
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[i][e] = 0.f;
  for (int kt = 0; kt < KT; ++kt) {
    const int stage = kt % RQ_STAGES;
    cp_async_wait<RQ_STAGES - 2>();
    __syncthreads();
    {
      const int nk = kt + RQ_STAGES - 1;
      if (nk < KT) load_b(nk, nk % RQ_STAGES);
      cp_async_commit();
    }
    const float* bs = Bs + stage * RQ_BK * RQ_BN;
    const int k0 = kt * RQ_BK;
#pragma unroll
    for (int kk = 0; kk < RQ_BK; kk += 4) {
      float4 a[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(rs + (warp + 8 * i) * RS + k0 + kk);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float4 b = *reinterpret_cast<const float4*>(bs + (kk + c) * RQ_BN + 4 * lane);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float av = c == 0 ? a[i].x : (c == 1 ? a[i].y : (c == 2 ? a[i].z : a[i].w));
          acc[i][0] = fmaf(av, b.x, acc[i][0]);
          acc[i][1] = fmaf(av, b.y, acc[i][1]);
          acc[i][2] = fmaf(av, b.z, acc[i][2]);
          acc[i][3] = fmaf(av, b.w, acc[i][3]);
        }
      }
    }
  }
  cp_async_wait<0>();

  // ---- distances + first-minimum argmin over this chunk
  const float4 en = *reinterpret_cast<const float4*>(p.enorm + c0 + 4 * lane);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = warp + 8 * i;
    const float xn = xnorm[r];
    float v = INFINITY;
    int idx = 0x7fffffff;
    const float en_e[4] = {en.x, en.y, en.z, en.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float d2 = (acc[i][e] + xn) + en_e[e];
      const float d = sqrtf(fmaxf(d2, 0.f));
      argmin_combine(v, idx, d, c0 + 4 * lane + e);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
      argmin_combine(v, idx, ov, oi);
    }
    const long long n = n0 + r;
    if (lane == 0 && n < p.N) {
      p.pval[n * p.nch + blockIdx.y] = v;
      p.pidx[n * p.nch + blockIdx.y] = idx;
    }
  }
}

// last level of a group: reduce partials -> code
__global__ void rvq_finish_kernel(const float* __restrict__ pval, const int* __restrict__ pidx, int nch,
                                  long long* __restrict__ codes, int level, long long N, int T, int n_q, int time_major) {
  const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float v = INFINITY;
  int idx = 0x7fffffff;
  for (int c = 0; c < nch; ++c) argmin_combine(v, idx, pval[n * nch + c], pidx[n * nch + c]);
  const long long nb = N / T;
  const long long b = time_major ? n % nb : n / T, t = time_major ? n / nb : n % T;
  codes[(b * n_q + level) * T + t] = idx;
}

// Sticky device-side error word (rstnet_device_error_flags): F.embedding raises on a code outside [0, bins); here the
// code is clamped (no out-of-bounds read) and bit 0 (1) is set.
__device__ unsigned int g_rvq_dev_err = 0;
unsigned int rvq_read_errors(bool clear) {
  unsigned int v = 0;
  cudaMemcpyFromSymbol(&v, g_rvq_dev_err, sizeof(v));
  if (clear && v) { const unsigned int z = 0; cudaMemcpyToSymbol(g_rvq_dev_err, &z, sizeof(z)); }
  return v;
}

// decode: q[n][0:dim) = sum_{l<ns} E_l[c_l];  q[n][dim:2dim) = sum_{l>=ns} E_l[c_l]  (level order)
__global__ void rvq_gather_kernel(const long long* __restrict__ codes, const float* __restrict__ E, float* __restrict__ q,
                                  long long N, int T, int n_q, int ns, int dim, int bins, int time_major) {
  const int d4n = dim / 4;
  const long long total = N * d4n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / d4n;
    const int d4 = (int)(i % d4n);
    const long long nb = N / T;
    const long long b = time_major ? n % nb : n / T, t = time_major ? n / nb : n % T;
    float4 s1 = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s1;
    for (int l = 0; l < n_q; ++l) {
      long long c = codes[(b * n_q + l) * T + t];
      if (c < 0 || c >= bins) {
        if (d4 == 0) atomicOr(&g_rvq_dev_err, 1u);
        c = c < 0 ? 0 : bins - 1;
      }
      const float4 e = *reinterpret_cast<const float4*>(E + ((long long)l * bins + c) * dim + 4 * d4);
      if (l < ns) { s1.x += e.x; s1.y += e.y; s1.z += e.z; s1.w += e.w; }
      else        { s2.x += e.x; s2.y += e.y; s2.z += e.z; s2.w += e.w; }
    }
    *reinterpret_cast<float4*>(q + n * 2 * dim + 4 * d4) = s1;
    *reinterpret_cast<float4*>(q + n * 2 * dim + dim + 4 * d4) = s2;
  }
}

static size_t rvq_smem_bytes(int dim) {
  return ((size_t)RQ_BM * (dim + 4) + 2 * RQ_BM + (size_t)RQ_STAGES * RQ_BK * RQ_BN) * sizeof(float);
}

}  // namespace rstnet
using namespace rstnet;

extern "C" int64_t rstnet_rvq_encode_workspace(int64_t N, int32_t n_q, int32_t dim, int32_t bins) {
  (void)n_q;
  const int64_t nch = (bins + RQ_BN - 1) / RQ_BN;
  // 2 groups x ping-pong residuals + 2 groups x ping-pong (pval + pidx)
  return 4 * N * dim * (int64_t)sizeof(float) + 4 * N * nch * (int64_t)(sizeof(float) + sizeof(int)) + 256;
}

extern "C" int rstnet_rvq_encode_f32(const float* x, int64_t ldx, const float* E, const float* Et, const float* enorm,
                                     int64_t* codes, void* work, int64_t N, int32_t T, int32_t n_q, int32_t ns,
                                     int32_t dim, int32_t bins, int32_t time_major, rstnet_stream_t stream) {
  RSTNET_REQUIRE(x && E && Et && enorm && codes && work, "rvq_encode: null pointer");
  RSTNET_REQUIRE(N > 0 && T > 0 && N % T == 0, "rvq_encode: N (%lld) must be a positive multiple of T (%d)", (long long)N, T);
  RSTNET_REQUIRE(n_q > 0 && ns >= 0 && ns <= n_q, "rvq_encode: bad level split");
  RSTNET_REQUIRE(dim % 16 == 0 && bins % RQ_BN == 0 && ldx % 4 == 0, "rvq_encode: dim %% 16, bins %% 128, ldx %% 4 required");
  // the level kernel reads x, the residuals, E and enorm as float4 and streams Et with 16-byte cp.async
  RSTNET_REQUIRE((uintptr_t)x % 16 == 0 && (uintptr_t)E % 16 == 0 && (uintptr_t)Et % 16 == 0 && (uintptr_t)enorm % 16 == 0 &&
                     (uintptr_t)work % 16 == 0 && (uintptr_t)codes % 8 == 0,
                 "rvq_encode: x, E, Et, enorm and work must be 16-byte aligned, codes 8-byte aligned");
  const size_t smem = rvq_smem_bytes(dim);
  RSTNET_REQUIRE(smem <= 220 * 1024, "rvq_encode: dim too large for shared memory");
  static unsigned long long attr = 0;
  smem_optin(rvq_level_kernel, 220 * 1024, attr);
  cudaStream_t st = (cudaStream_t)stream;
  const int nch = bins / RQ_BN;
  char* w = (char*)work;
  float* R[2][2];
  for (int g = 0; g < 2; ++g)
    for (int i = 0; i < 2; ++i) { R[g][i] = (float*)w; w += (size_t)N * dim * sizeof(float); }
  // partial minima are ping-ponged too: a level's CTAs read the previous level's partials while
  // sibling CTAs (other centroid chunks of the same frames) are already writing this level's
  float* PV[2][2]; int* PI[2][2];
  for (int g = 0; g < 2; ++g)
    for (int i = 0; i < 2; ++i) { PV[g][i] = (float*)w; w += (size_t)N * nch * sizeof(float); }
  for (int g = 0; g < 2; ++g)
    for (int i = 0; i < 2; ++i) { PI[g][i] = (int*)w; w += (size_t)N * nch * sizeof(int); }
  dim3 grid((unsigned)ceil_div(N, RQ_BM), (unsigned)nch);
  for (int g = 0; g < 2; ++g) {
    const int l0 = g == 0 ? 0 : ns, l1 = g == 0 ? ns : n_q;
    for (int l = l0; l < l1; ++l) {
      RvqLevelParams p;
      const int j = l - l0;
      p.x_first = j == 0 ? x + (g == 0 ? 0 : dim) : nullptr;
      p.ldx = ldx;
      p.r_prev = R[g][(j + 1) & 1];
      p.r_cur = R[g][j & 1];
      p.e_prev = j == 0 ? nullptr : E + (size_t)(l - 1) * bins * dim;
      p.pval_prev = PV[g][(j + 1) & 1];
      p.pidx_prev = PI[g][(j + 1) & 1];
      p.codes = (long long*)codes;
      p.prev_level = l - 1;
      p.et = Et + (size_t)l * dim * bins;
      p.enorm = enorm + (size_t)l * bins;
      p.pval = PV[g][j & 1];
      p.pidx = PI[g][j & 1];
      p.N = N; p.T = T; p.n_q = n_q; p.dim = dim; p.bins = bins; p.nch = nch; p.time_major = time_major;
      rvq_level_kernel<<<grid, RQ_NT, smem, st>>>(p);
      count_launch();
      if (int e = check_launch("rvq_level")) return e;
    }
    if (l1 > l0) {
      const int jl = (l1 - 1 - l0) & 1;
      rvq_finish_kernel<<<ceil_div(N, 256), 256, 0, st>>>(PV[g][jl], PI[g][jl], nch, (long long*)codes, l1 - 1, N, T, n_q, time_major);
      count_launch();
      if (int e = check_launch("rvq_finish")) return e;
    }
  }
  return 0;
}

extern "C" int rstnet_rvq_decode_gather_f32(const int64_t* codes, const float* E, float* q, int64_t N, int32_t T,
                                            int32_t n_q, int32_t ns, int32_t dim, int32_t bins, int32_t time_major,
                                            rstnet_stream_t stream) {
  RSTNET_REQUIRE(codes && E && q, "rvq_decode_gather: null pointer");
  RSTNET_REQUIRE(N > 0 && T > 0 && N % T == 0 && dim % 4 == 0, "rvq_decode_gather: bad shape");
  RSTNET_REQUIRE((uintptr_t)E % 16 == 0 && (uintptr_t)q % 16 == 0 && (uintptr_t)codes % 8 == 0,
                 "rvq_decode_gather: E and q must be 16-byte aligned, codes 8-byte aligned");
  const long long total = (long long)N * (dim / 4);
  int gx = ceil_div(total, 256);
  if (gx > sm_count() * 16) gx = sm_count() * 16;
  rvq_gather_kernel<<<gx, 256, 0, (cudaStream_t)stream>>>((const long long*)codes, E, q, N, T, n_q, ns, dim, bins, time_major);
  count_launch();
  return check_launch("rvq_decode_gather");
}
