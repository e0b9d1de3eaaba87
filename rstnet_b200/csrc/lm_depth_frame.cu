// The depth transformer of one frame as ONE persistent kernel (SURVEY.md H5): up to dep_q codebook steps x 6 layers of
// per-step weights, <= 8 keys of attention per step, and the token sampling between steps, all inside a single
// cooperative launch -- instead of ~50 launches per step (4 skinny GEMMs + 3 finalizes + attention per layer, sampler,
// embedding gather).  Reference: GPT.forward_codecformer (models/llama_streaming.py:727-749) over the
// StreamingTransformer with weights_per_step (modules/transformer.py:155-179, 375-419, 518-577), ActivationGating
// (modules/gating.py:12-21), sample_token* (utils/sampling.py:85-154).
//
// Why this shape: a step streams only 2-11 MB of weights per GEMM (1.27 GB per frame = 0.38 ms at the H100 data-sheet 3.35 TB/s) and the
// eight steps are sequentially dependent, so the frame is bound by per-launch fixed costs, not by bandwidth or math.
// Here every SM stays resident; a GEMM phase gives each CTA a few 16-row blocks of the weight matrix, which it streams
// once through a 3-stage cp.async ring while the (tiny) activation panel [M <= 128 streams][K] comes from L2; the
// contraction runs on mma.sync (bf16, fp32 accumulate) -- the tensor pipe is idle either way at M <= 128 and a
// register-operand MMA needs no shared-memory descriptor set-up per phase.  Phases are separated by a grid-wide barrier
// (one atomic per CTA).  RMSNorm is folded into the consumer: the producer's epilogue leaves per-block sums of squares,
// the consumer scales the activation fragments on the fly (same fp32 arithmetic as modules/transformer.py:34-48).
// bf16 roundings follow the eager reference: a linear's output is rounded before the residual / embedding add.
#include <cuda_bf16.h>

#include <cstdlib>

#include "common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {
extern void count_launch();
typedef __nv_bfloat16 bf16;
namespace {
__device__ __forceinline__ float b2f(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ bf16 f2b(float v) { return __float2bfloat16(v); }
#include "lm_sample.cuh"
}  // namespace

constexpr int DF_THREADS = 256;
constexpr int DF_KC = 128;                // K elements per pipeline stage
constexpr int DF_PITCH = DF_KC * 2 + 16;  // shared-memory row pitch in bytes: 8 consecutive rows hit distinct banks (ldmatrix)
// pipeline depth: per chunk a CTA has only ~30 KB in flight, and a chunk costs a full DRAM round trip (with 3 stages the
// phases ran at memory latency); 6 stages for <= 64 streams, 4 for <= 128 (shared-memory budget)
constexpr int DF_MAXU = 3;                // 16-row weight blocks per CTA per round
constexpr int DF_MAXQ = 8, DF_MAXL = 8;
constexpr int DF_SMEM_MAX = 201 * 1024;   // dynamic; the sampler's static arrays (25 KB) come on top: 227 KB per CTA in all

struct DepthFrameParams {
  int M, D, E, Hp, H, hd, Q, L, card;
  int k_begin, k_end, ring_quirk, do_sample;
  const bf16* tout;      // [M][E] transformer_out
  const bf16* emb0_rows; // optional [M][D]: the step-0 input embedding as features (forward_local) instead of a token id
  bf16* x;               // [M][D] residual stream
  bf16* qkv;             // [M][3][H][hd]
  bf16* att;             // [M][D]
  bf16* dh;              // [M][Hp]
  bf16* logits;          // [Q][M][card]: one buffer per step (an address is written once per launch: no stale L1 lines)
  bf16* dkv;             // [L][2][M][H][Q][hd]
  float* ss_part;        // [D/16][M] sums of squares of x per 16-column block
  long long* tokens;     // [M][tok_stride]: column k = input token of step k, column k + 1 = its output
  int tok_stride;
  unsigned int* barrier; // zeroed by the host before every launch
  unsigned int* err;     // sticky error word (bit 0 bad token id, bit 2 barrier timeout)
  const bf16* w_in[DF_MAXQ];          // codecformer_in[k]            [D][E]
  const bf16* emb[DF_MAXQ];           // embedding table of step k     [emb_rows][D]
  long long emb_rows[DF_MAXQ];
  const bf16* w_qkv[DF_MAXL];         // in_proj_weight                [Q*3D][D]
  const bf16* w_out[DF_MAXL];         // out_proj.weight               [Q*D][D]
  const bf16* a1[DF_MAXL];
  const bf16* a2[DF_MAXL];
  const bf16* w_gin[DF_MAXL][DF_MAXQ];   // gating linear_in, rows interleaved in 8-row groups [a(8); b(8)]  [2*Hp][D]
  const bf16* w_gout[DF_MAXL][DF_MAXQ];  // gating linear_out, K padded    [D][Hp]
  const bf16* w_head[DF_MAXQ];        // audio_linears[k]              [card][D]
  int top_k; float temp; unsigned int seed; const long long* frame_counter; int n_valid[DF_MAXQ];
  int dbg;               // profiling aid (RSTNET_DEPTH_DBG): bit 0 skip the MMA loop, bit 1 skip the cp.async loads, bit 2 skip the epilogue
  long long* trace;      // profiling aid (RSTNET_DEPTH_TRACE): CTA 0 stamps clock64 after every phase and every barrier
};

#define DF_STAMP()                                                      \
  do {                                                                  \
    if (p.trace && blockIdx.x == 0 && threadIdx.x == 0) p.trace[tr++] = clock64(); \
  } while (0)

__device__ __forceinline__ void cp_async16_cg(uint32_t smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_dst), "l"(gsrc));
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldmatrix_x2(uint32_t addr, uint32_t& r0, uint32_t& r1) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0,%1}, [%2];\n" : "=r"(r0), "=r"(r1) : "r"(addr));
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t scale_pair(uint32_t v, float s0, float s1) {
  // two bf16 activations -> bf16(x * (alpha * r)) each: the fp32 arithmetic of _rms_norm (modules/transformer.py:44-47)
  const __nv_bfloat162 in = *reinterpret_cast<const __nv_bfloat162*>(&v);
  const float2 f = __bfloat1622float2(in);
  const __nv_bfloat162 out = __floats2bfloat162_rn(f.x * s0, f.y * s1);
  return *reinterpret_cast<const uint32_t*>(&out);
}

// grid-wide barrier: one arrival per CTA on a monotonically growing counter (zeroed by the host before the launch).
// The launch is cooperative, so all CTAs are resident; the spin still carries a watchdog so that a lost CTA shows up as
// an error flag and garbage output instead of a hung device.
__device__ __forceinline__ void grid_barrier(const DepthFrameParams& p, unsigned int& target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    __threadfence();
    atomicAdd(p.barrier, 1u);
    const long long t0 = clock64();
    unsigned int spins = 0;
    while (true) {
      unsigned int v;
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p.barrier) : "memory");
      if (v >= target) break;
      if ((++spins & 1023u) == 0) {
        unsigned int e;
        asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(e) : "l"(p.err) : "memory");
        if (e & 4u) break;                                                    // somebody already gave up: do not wait again
        if (clock64() - t0 > 2000000000LL) { atomicOr(p.err, 4u); break; }   // ~1 s
      }
    }
    __threadfence();
  }
  __syncthreads();
}

enum DfEpi : int { EPI_STORE = 0, EPI_RES = 1, EPI_IN = 2, EPI_SILU = 3 };

// out[m][n] (op)= sum_k Xs[m][k] * W[n][k]; every CTA takes the 16-row weight blocks u = blockIdx.x + j * gridDim.x.
//   norm_alpha != nullptr: Xs[m][k] = bf16(X[m][k] * (alpha[k] * r[m])), r[m] = rsqrt(1e-8 + sum_j ss_part[j][m] / K)
//   EPI_STORE: out = bf16(acc)                                   (qkv, logits)
//   EPI_RES:   out = bf16(bf16(acc) + out)  + ss_part             (out-proj / gating-out residual adds)
//   EPI_IN:    out = bf16(bf16(acc) + emb[token[m]])  + ss_part   (step input: codecformer_in + token embedding)
//   EPI_SILU:  rows [a(8); b(8)] per block: out[m][8u+g] = bf16(bf16(silu(bf16 a)) * bf16 b)
// issue the weight chunks 0 .. STAGES-2 of a phase's first round (one cp.async group each) -- they do not depend on the
// previous phase, so they are put in flight BEFORE the grid barrier that precedes the phase
template <int STAGES>
__device__ void prefetch_weights(const DepthFrameParams& p, uint8_t* smem, const bf16* __restrict__ W, int N, int K) {
  const int Mpad = (p.M + 7) & ~7;
  const int x_bytes = Mpad * DF_PITCH, stage_bytes = x_bytes + DF_MAXU * 16 * DF_PITCH;
  const uint32_t smem_base = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
  const int nunits = (N + 15) / 16, nchunks = K / DF_KC;
  int U = 0;
  int units[DF_MAXU];
#pragma unroll
  for (int i = 0; i < DF_MAXU; ++i) {
    units[i] = blockIdx.x + i * gridDim.x;
    if (units[i] < nunits) U = i + 1;
  }
  for (int c = 0; c < STAGES - 1; ++c) {
    if (c < nchunks) {
      const uint32_t ws = smem_base + (c % STAGES) * stage_bytes + x_bytes;
      for (int i = threadIdx.x; i < U * 256; i += DF_THREADS) {
        const int ui = i >> 8, r = (i >> 4) & 15, piece = i & 15;
        int n = units[ui] * 16 + r;
        n = n < N ? n : N - 1;
        cp_async16_cg(ws + (ui * 16 + r) * DF_PITCH + piece * 16, W + (long long)n * K + c * DF_KC + piece * 8);
      }
    }
    cp_async_commit();
  }
}

template <int EPI, int STAGES>
__device__ void gemm_phase(const DepthFrameParams& p, uint8_t* smem, const bf16* __restrict__ W, int N, int K,
                           const bf16* __restrict__ X, int ldx, const bf16* __restrict__ norm_alpha, bf16* __restrict__ out, int ldo,
                           int step_k, bool w_prefetched) {
  const int M = p.M;
  const int tid = threadIdx.x, warp = tid / 32, lane = tid % 32;
  const int Mpad = (M + 7) & ~7;
  const int x_bytes = Mpad * DF_PITCH;
  const int stage_bytes = x_bytes + DF_MAXU * 16 * DF_PITCH;
  float* s_r = reinterpret_cast<float*>(smem + STAGES * stage_bytes);   // [128]
  float* s_alpha = s_r + 128;                                                // [K] (norm phases have K == D)
  const int nunits = (N + 15) / 16;
  const int nchunks = K / DF_KC;
  const uint32_t smem_base = static_cast<uint32_t>(__cvta_generic_to_shared(smem));

  if (norm_alpha) {
    // r[m] from the producer's per-block sums of squares.  The nb partials of a row are spread over `nsub` threads, each
    // issuing its loads in independent batches of 8 (a plain dependent loop costs nb L2 round trips per phase),
    // then added in a fixed order.
    const int nb = K / 16;
    const int mc = Mpad <= 64 ? 64 : 128, nsub = DF_THREADS / mc;
    const int m = tid % mc, q = tid / mc;
    float ss = 0.f;
    if (m < M) {
      for (int j0 = q; j0 < nb; j0 += 8 * nsub) {
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int j = j0 + e * nsub;
          v[e] = j < nb ? __ldcg(p.ss_part + (long long)j * M + m) : 0.f;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) ss += v[e];
      }
    }
    s_alpha[q * 128 + m] = ss;            // scratch: [nsub][128] partial sums (the buffer holds max(D, 512) floats)
    __syncthreads();
    if (tid < Mpad) {
      float tot = 0.f;
      for (int qq = 0; qq < nsub; ++qq) tot += s_alpha[qq * 128 + tid];
      s_r[tid] = rsqrtf(1e-8f + tot / (float)K);
    }
    __syncthreads();
    for (int k = tid; k < K; k += DF_THREADS) s_alpha[k] = b2f(norm_alpha[k]);
  }
  __syncthreads();

  for (int u0 = blockIdx.x; u0 < nunits; u0 += gridDim.x * DF_MAXU) {
    int U = 0;
    int units[DF_MAXU];
#pragma unroll
    for (int i = 0; i < DF_MAXU; ++i) {
      units[i] = u0 + i * gridDim.x;
      if (units[i] < nunits) U = i + 1;
    }
    auto issue = [&](int c, bool with_w) {
      if (p.dbg & 2) { cp_async_commit(); return; }
      const int s = c % STAGES;
      const uint32_t xs = smem_base + s * stage_bytes, ws = xs + x_bytes;
      const int k0 = c * DF_KC;
      for (int i = tid; i < Mpad * 16; i += DF_THREADS) {       // 16 x 16-byte pieces per 128-element row
        const int m = i >> 4, piece = i & 15;
        const int mm = m < M ? m : M - 1;                       // padding rows repeat the last stream (never stored)
        cp_async16_cg(xs + m * DF_PITCH + piece * 16, X + (long long)mm * ldx + k0 + piece * 8);
      }
      if (with_w) {
        for (int i = tid; i < U * 256; i += DF_THREADS) {
          const int ui = i >> 8, r = (i >> 4) & 15, piece = i & 15;
          int n = units[ui] * 16 + r;
          n = n < N ? n : N - 1;
          cp_async16_cg(ws + (ui * 16 + r) * DF_PITCH + piece * 16, W + (long long)n * K + k0 + piece * 8);
        }
      }
      cp_async_commit();
    };
    const bool pre = w_prefetched && u0 == (int)blockIdx.x;    // the first round's first weight chunks are already in flight
    float acc[DF_MAXU][2][4];
#pragma unroll
    for (int i = 0; i < DF_MAXU; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

    for (int c = 0; c < STAGES - 1; ++c) {
      if (c < nchunks) issue(c, !pre); else cp_async_commit();
    }
    for (int c = 0; c < nchunks; ++c) {
      cp_async_wait<STAGES - 2>();
      __syncthreads();                       // chunk c landed for everyone; everyone is done with chunk c - 1's slot
      if (c + STAGES - 1 < nchunks) issue(c + STAGES - 1, true); else cp_async_commit();
      const int s = c % STAGES;
      const uint32_t xs = smem_base + s * stage_bytes, ws = xs + x_bytes;
      const int k0 = c * DF_KC;
      if (p.dbg & 1) continue;
#pragma unroll
      for (int ks = 0; ks < DF_KC / 16; ++ks) {
        uint32_t bfrag[2][2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int nt = warp + 8 * j;
          if (nt * 8 < Mpad) {
            ldmatrix_x2(xs + (nt * 8 + (lane & 7)) * DF_PITCH + (ks * 16 + ((lane >> 3) & 1) * 8) * 2, bfrag[j][0], bfrag[j][1]);
            if (norm_alpha) {
              const float r = s_r[nt * 8 + (lane >> 2)];
              const int kk = k0 + ks * 16 + (lane & 3) * 2;
              bfrag[j][0] = scale_pair(bfrag[j][0], s_alpha[kk] * r, s_alpha[kk + 1] * r);
              bfrag[j][1] = scale_pair(bfrag[j][1], s_alpha[kk + 8] * r, s_alpha[kk + 9] * r);
            }
          }
        }
#pragma unroll
        for (int i = 0; i < DF_MAXU; ++i) {
          if (i < U) {
            uint32_t a[4];
            ldmatrix_x4(ws + (i * 16 + (lane & 7) + ((lane >> 3) & 1) * 8) * DF_PITCH + (ks * 16 + (lane >> 4) * 8) * 2, a[0], a[1], a[2], a[3]);
#pragma unroll
            for (int j = 0; j < 2; ++j)
              if ((warp + 8 * j) * 8 < Mpad) mma_bf16_16816(acc[i][j], a, bfrag[j][0], bfrag[j][1]);
          }
        }
      }
    }
    cp_async_wait<0>();
    __syncthreads();                         // all warps done with the last stages before the next round refills them

    // ---- epilogue: thread holds rows g, g + 8 of the block and streams 2t, 2t + 1 of its n-tile
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int i = 0; i < DF_MAXU; ++i) {
      if (i >= U || (p.dbg & 4)) continue;
      const int u = units[i];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int nt = warp + 8 * j;
        if (nt * 8 >= Mpad) continue;
        const int m0 = nt * 8 + 2 * t;
        const float* d = acc[i][j];
        if (EPI == EPI_SILU) {
          const int c = u * 8 + g;           // gating column; row g is a_c, row g + 8 is b_c
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int m = m0 + e;
            if (m < M) {
              const float a = b2f(f2b(d[e])), b = b2f(f2b(d[2 + e]));
              const float sl = b2f(f2b(a / (1.0f + expf(-a))));
              out[(long long)m * ldo + c] = f2b(sl * b);
            }
          }
        } else {
          float sq[2] = {0.f, 0.f};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int n = u * 16 + g + (e >> 1) * 8, m = m0 + (e & 1);
            if (n < N && m < M) {
              bf16* o = out + (long long)m * ldo + n;
              float v = b2f(f2b(d[e]));
              if (EPI == EPI_RES) {
                const bf16 rv = __ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(o)));   // L2: no stale L1 line
                v = b2f(f2b(v + b2f(rv)));
              } else if (EPI == EPI_IN) {
                float ev = 0.f;
                if (step_k == 0 && p.emb0_rows) {
                  ev = b2f(p.emb0_rows[(long long)m * p.D + n]);      // forward_local hands the step-0 embedding in as features
                } else {
                  const long long id = __ldcg(p.tokens + (long long)m * p.tok_stride + step_k);
                  if (id < -1 || id >= p.emb_rows[step_k]) { ev = __int_as_float(0x7fc00000); atomicOr(p.err, 1u); }
                  else if (id >= 0) ev = b2f(p.emb[step_k][id * p.D + n]);
                }
                v = b2f(f2b(v + ev));
              }
              *o = f2b(v);
              if (EPI != EPI_STORE) sq[e & 1] = fmaf(v, v, sq[e & 1]);
            }
          }
          if (EPI != EPI_STORE) {
            // sum of squares of this block's 16 columns per stream: reduce over the 8 row groups (lane bits 2..4)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float s = sq[e];
              s += __shfl_xor_sync(0xffffffffu, s, 4);
              s += __shfl_xor_sync(0xffffffffu, s, 8);
              s += __shfl_xor_sync(0xffffffffu, s, 16);
              if (g == 0 && m0 + e < M) p.ss_part[(long long)u * M + m0 + e] = s;
            }
          }
        }
      }
    }
  }
}

// one warp per (stream, head): append this step's k, v at slot `step`, attend keys j_lo..step (<= 8 keys)
__device__ void attention_phase(const DepthFrameParams& p, int layer, int step) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int H = p.H, hd = p.hd, HD = H * hd, cap = p.Q;
  const float scale = rsqrtf((float)hd);
  const int j_lo = (p.ring_quirk && step + 2 - cap > 0) ? step + 2 - cap : 0;   // RingKVCache.complete's labelling (transformer.py:258-263)
  for (int item = blockIdx.x * (DF_THREADS / 32) + warp; item < p.M * H; item += gridDim.x * (DF_THREADS / 32)) {
    const int m = item / H, h = item % H;
    const bf16* qp = p.qkv + (long long)m * 3 * HD + h * hd;
    bf16* Kb = p.dkv + ((((long long)layer * 2) * p.M + m) * H + h) * cap * hd;
    bf16* Vb = Kb + (long long)p.M * H * cap * hd;
    float qv[4], kn[4], vn[4];            // hd <= 128: up to 4 dims per lane
    const int nd = (hd + 31) / 32;
    for (int i = 0; i < nd; ++i) {
      const int dd = lane + 32 * i;
      if (dd < hd) {
        qv[i] = b2f(__ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(qp + dd))));
        const bf16 kx = __ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(qp + HD + dd)));
        const bf16 vx = __ushort_as_bfloat16(__ldcg(reinterpret_cast<const unsigned short*>(qp + 2 * HD + dd)));
        Kb[(long long)step * hd + dd] = kx;
        Vb[(long long)step * hd + dd] = vx;
        kn[i] = b2f(kx); vn[i] = b2f(vx);
      } else { qv[i] = 0.f; kn[i] = 0.f; vn[i] = 0.f; }
    }
    float sc[8];
    float mx = -INFINITY;
    for (int j = j_lo; j <= step; ++j) {
      float dot = 0.f;
      for (int i = 0; i < nd; ++i) {
        const int dd = lane + 32 * i;
        if (dd < hd) dot = fmaf(qv[i], j == step ? kn[i] : b2f(Kb[(long long)j * hd + dd]), dot);
      }
      dot = warp_sum(dot) * scale;
      sc[j] = dot;
      mx = fmaxf(mx, dot);
    }
    float l = 0.f;
    for (int j = j_lo; j <= step; ++j) { sc[j] = __expf(sc[j] - mx); l += sc[j]; }
    for (int i = 0; i < nd; ++i) {
      const int dd = lane + 32 * i;
      if (dd < hd) {
        float a = 0.f;
        for (int j = j_lo; j <= step; ++j) a = fmaf(sc[j], j == step ? vn[i] : b2f(Vb[(long long)j * hd + dd]), a);
        p.att[(long long)m * HD + h * hd + dd] = f2b(a / l);
      }
    }
  }
}

template <int STAGES>
__global__ void __launch_bounds__(DF_THREADS, 1) depth_frame_kernel(const __grid_constant__ DepthFrameParams p) {
  extern __shared__ __align__(128) uint8_t df_smem[];
  unsigned int target = 0;
  int tr = 0;
  const int D = p.D;
  DF_STAMP();
  bool pf = false;    // the next GEMM phase's first weight chunks are already in flight
  for (int k = p.k_begin; k < p.k_end; ++k) {
    gemm_phase<EPI_IN, STAGES>(p, df_smem, p.w_in[k], D, p.E, p.tout, p.E, nullptr, p.x, D, k, pf);
    prefetch_weights<STAGES>(p, df_smem, p.w_qkv[0] + (long long)k * 3 * D * D, 3 * D, D);
    DF_STAMP(); grid_barrier(p, target); DF_STAMP();
    for (int l = 0; l < p.L; ++l) {
      gemm_phase<EPI_STORE, STAGES>(p, df_smem, p.w_qkv[l] + (long long)k * 3 * D * D, 3 * D, D, p.x, D, p.a1[l], p.qkv, 3 * D, k, true);
      prefetch_weights<STAGES>(p, df_smem, p.w_out[l] + (long long)k * D * D, D, D);      // in flight across the attention phase
      DF_STAMP(); grid_barrier(p, target); DF_STAMP();
      attention_phase(p, l, k);
      DF_STAMP(); grid_barrier(p, target); DF_STAMP();
      gemm_phase<EPI_RES, STAGES>(p, df_smem, p.w_out[l] + (long long)k * D * D, D, D, p.att, D, nullptr, p.x, D, k, true);
      prefetch_weights<STAGES>(p, df_smem, p.w_gin[l][k], 2 * p.Hp, D);
      DF_STAMP(); grid_barrier(p, target); DF_STAMP();
      gemm_phase<EPI_SILU, STAGES>(p, df_smem, p.w_gin[l][k], 2 * p.Hp, D, p.x, D, p.a2[l], p.dh, p.Hp, k, true);
      prefetch_weights<STAGES>(p, df_smem, p.w_gout[l][k], D, p.Hp);
      DF_STAMP(); grid_barrier(p, target); DF_STAMP();
      gemm_phase<EPI_RES, STAGES>(p, df_smem, p.w_gout[l][k], D, p.Hp, p.dh, p.Hp, nullptr, p.x, D, k, true);
      if (l + 1 < p.L) prefetch_weights<STAGES>(p, df_smem, p.w_qkv[l + 1] + (long long)k * 3 * D * D, 3 * D, D);
      else prefetch_weights<STAGES>(p, df_smem, p.w_head[k], p.card, D);
      DF_STAMP(); grid_barrier(p, target); DF_STAMP();
    }
    bf16* lg = p.logits + (long long)k * p.M * p.card;
    gemm_phase<EPI_STORE, STAGES>(p, df_smem, p.w_head[k], p.card, D, p.x, D, nullptr, lg, p.card, k, true);
    pf = false;
    if (k + 1 < p.k_end) { prefetch_weights<STAGES>(p, df_smem, p.w_in[k + 1], D, p.E); pf = true; }
    DF_STAMP();
    if (p.do_sample || k + 1 < p.k_end) grid_barrier(p, target);     // logits complete; nobody still reads x
    DF_STAMP();
    if (p.do_sample) {
      const unsigned int stepc = p.frame_counter ? (unsigned int)(*p.frame_counter) : 0u;
      for (int m = blockIdx.x; m < p.M; m += gridDim.x)
        sample_row(lg + (long long)m * p.card, p.n_valid[k], p.top_k, p.temp, p.seed + (unsigned int)(k + 1), stepc, m,
                   p.tokens + (long long)m * p.tok_stride + k + 1);
      if (k + 1 < p.k_end) grid_barrier(p, target);                  // the sampled tokens feed the next step's embedding
    }
  }
  cp_async_wait<0>();
}

}  // namespace rstnet
using namespace rstnet;

struct rstnet_depth_plan {
  DepthFrameParams p;
  int grid;
  int stages;
  size_t smem;
  long long* trace = nullptr;
};

extern "C" void rstnet_lm_depth_frame_set_trace(rstnet_depth_plan* pl, int64_t* trace) { pl->trace = (long long*)trace; }

extern "C" int rstnet_lm_depth_frame_create(const rstnet_depth_frame_desc* d, rstnet_depth_plan** out) {
  RSTNET_REQUIRE(d && out, "depth_frame_create: null pointer");
  RSTNET_REQUIRE(d->M >= 1 && d->M <= 128, "depth_frame_create: 1 <= M <= 128 (got %d)", d->M);
  RSTNET_REQUIRE(d->Q >= 1 && d->Q <= DF_MAXQ && d->L >= 1 && d->L <= DF_MAXL, "depth_frame_create: dep_q <= 8, layers <= 8");
  RSTNET_REQUIRE(d->D % DF_KC == 0 && d->E % DF_KC == 0 && d->Hp % DF_KC == 0 && d->D <= 2048,
                 "depth_frame_create: D, E, padded gating width must be multiples of %d, D <= 2048 (D=%d E=%d Hp=%d)", DF_KC, d->D, d->E, d->Hp);
  RSTNET_REQUIRE(d->H * d->hd == d->D && d->hd <= 128, "depth_frame_create: heads * head_dim must equal D, head_dim <= 128");
  rstnet_depth_plan* pl = new rstnet_depth_plan();
  DepthFrameParams& p = pl->p;
  p.M = d->M; p.D = d->D; p.E = d->E; p.Hp = d->Hp; p.H = d->H; p.hd = d->hd; p.Q = d->Q; p.L = d->L; p.card = d->card;
  p.k_begin = 0; p.k_end = d->Q; p.ring_quirk = 1; p.do_sample = 0;
  p.emb0_rows = nullptr;
  p.tout = (const bf16*)d->tout; p.x = (bf16*)d->x; p.qkv = (bf16*)d->qkv; p.att = (bf16*)d->att; p.dh = (bf16*)d->dh;
  p.logits = (bf16*)d->logits; p.dkv = (bf16*)d->dkv; p.ss_part = d->ss_part; p.tokens = (long long*)d->tokens;
  p.tok_stride = d->tok_stride; p.barrier = (unsigned int*)d->barrier; p.err = (unsigned int*)d->barrier + 1;
  for (int k = 0; k < d->Q; ++k) {
    p.w_in[k] = (const bf16*)d->w_in[k]; p.emb[k] = (const bf16*)d->emb[k]; p.emb_rows[k] = d->emb_rows[k];
    p.w_head[k] = (const bf16*)d->w_head[k];
    RSTNET_REQUIRE(p.w_in[k] && p.emb[k] && p.w_head[k], "depth_frame_create: null weight pointer (step %d)", k);
  }
  for (int l = 0; l < d->L; ++l) {
    p.w_qkv[l] = (const bf16*)d->w_qkv[l]; p.w_out[l] = (const bf16*)d->w_out[l];
    p.a1[l] = (const bf16*)d->a1[l]; p.a2[l] = (const bf16*)d->a2[l];
    for (int k = 0; k < d->Q; ++k) {
      p.w_gin[l][k] = (const bf16*)d->w_gin[l * d->Q + k];
      p.w_gout[l][k] = (const bf16*)d->w_gout[l * d->Q + k];
      RSTNET_REQUIRE(p.w_gin[l][k] && p.w_gout[l][k], "depth_frame_create: null gating weight (layer %d step %d)", l, k);
    }
  }
  p.top_k = 0; p.temp = 1.f; p.seed = 0; p.frame_counter = nullptr; p.trace = nullptr; p.dbg = 0;
  for (int k = 0; k < DF_MAXQ; ++k) p.n_valid[k] = d->card;
  const int Mpad = (d->M + 7) & ~7;
  pl->stages = d->M <= 64 ? 6 : 4;
  pl->smem = (size_t)pl->stages * (Mpad * DF_PITCH + DF_MAXU * 16 * DF_PITCH) + 128 * sizeof(float) +
             (size_t)(d->D > 512 ? d->D : 512) * sizeof(float);      // s_alpha doubles as a [4][128] reduction scratch
  RSTNET_REQUIRE(pl->smem <= DF_SMEM_MAX, "depth_frame_create: shared memory budget exceeded");
  static unsigned long long attr6 = 0, attr4 = 0;
  if (pl->stages == 6) smem_optin(depth_frame_kernel<6>, DF_SMEM_MAX, attr6); else smem_optin(depth_frame_kernel<4>, DF_SMEM_MAX, attr4);
  int dev = 0, sms = 0, per_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (pl->stages == 6) cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, depth_frame_kernel<6>, DF_THREADS, pl->smem);
  else cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, depth_frame_kernel<4>, DF_THREADS, pl->smem);
  if (per_sm < 1) { delete pl; set_error("depth_frame_create: the kernel does not fit on an SM"); return 3; }
  pl->grid = sms;
  *out = pl;
  return 0;
}

extern "C" int rstnet_lm_depth_frame_run(const rstnet_depth_plan* pl, int32_t k_begin, int32_t k_end, int32_t ring_quirk, int32_t do_sample,
                                         int32_t top_k, float temp, uint32_t seed, const int64_t* frame_counter, const int32_t* n_valid,
                                         const void* step0_embedding, rstnet_stream_t stream) {
  RSTNET_REQUIRE(pl != nullptr, "depth_frame_run: null plan");
  RSTNET_REQUIRE(k_begin >= 0 && k_begin < k_end && k_end <= pl->p.Q, "depth_frame_run: bad step range [%d, %d)", k_begin, k_end);
  RSTNET_REQUIRE(!do_sample || (top_k <= SAMPLE_CAND && (top_k == 0 || temp > 0.f)), "depth_frame_run: bad sampling parameters");
  static unsigned long long attr6 = 0, attr4 = 0;           // per device (create may have run with another device current)
  if (pl->stages == 6) smem_optin(depth_frame_kernel<6>, DF_SMEM_MAX, attr6); else smem_optin(depth_frame_kernel<4>, DF_SMEM_MAX, attr4);
  DepthFrameParams p = pl->p;
  p.k_begin = k_begin; p.k_end = k_end; p.ring_quirk = ring_quirk; p.do_sample = do_sample;
  p.top_k = top_k; p.temp = temp; p.seed = seed; p.frame_counter = (const long long*)frame_counter;
  p.emb0_rows = (const bf16*)step0_embedding;
  p.trace = pl->trace;
  { const char* e = getenv("RSTNET_DEPTH_DBG"); p.dbg = e ? atoi(e) : 0; }
  for (int k = 0; k < pl->p.Q; ++k) {
    int nv = n_valid ? n_valid[k] : p.card;
    if (nv <= 0 || nv > p.card) nv = p.card;
    p.n_valid[k] = nv;
  }
  if (p.top_k > 0) for (int k = 0; k < pl->p.Q; ++k) if (p.top_k > p.n_valid[k]) p.top_k = p.n_valid[k];
  cudaStream_t st = (cudaStream_t)stream;
  cudaMemsetAsync(p.barrier, 0, sizeof(unsigned int), st);   // the arrival counter; the error word next to it is sticky
  void* args[] = {(void*)&p};
  const void* fn = pl->stages == 6 ? (const void*)depth_frame_kernel<6> : (const void*)depth_frame_kernel<4>;
  cudaError_t e = cudaLaunchCooperativeKernel(fn, dim3(pl->grid), dim3(DF_THREADS), args, pl->smem, st);
  count_launch();
  if (e != cudaSuccess) {
    set_error("depth_frame_run: cooperative launch failed: %s", cudaGetErrorString(e));
    return 2;
  }
  return check_launch("depth_frame");
}

extern "C" void rstnet_lm_depth_frame_destroy(rstnet_depth_plan* pl) { delete pl; }
