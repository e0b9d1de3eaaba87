// HBM-bound bf16 kernels of the speech-text LM decode step: embedding sum, RMSNorm (two variants),
// rotate-half RoPE + ring-KV append, ring decode attention, SiLU gating, depth-transformer attention,
// embedding gather, greedy / top-k sampling.  One token per stream (T == 1): rows are streams.
#include <cuda_bf16.h>

#include <cstdlib>
#include "common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {
extern void count_launch();
typedef __nv_bfloat16 bf16;

// Sticky device-side error word (include/rstnet_b200.h: rstnet_device_error_flags): kernels cannot raise, so an
// out-of-range id / position poisons its output and sets a bit the host reads at its next check.
__device__ unsigned int g_lm_dev_err = 0;
unsigned int lm_read_errors(bool clear) {
  unsigned int v = 0;
  cudaMemcpyFromSymbol(&v, g_lm_dev_err, sizeof(v));
  if (clear && v) { const unsigned int z = 0; cudaMemcpyToSymbol(g_lm_dev_err, &z, sizeof(z)); }
  return v;
}

__device__ __forceinline__ float b2f(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ bf16 f2b(float v) { return __float2bfloat16(v); }

// ---------------------------------------------------------------- embedding sum (llama_streaming.py:680-687)
// x[b] = ((e_0 + e_1) + ... + e_{nq-1}) + wte[text]; every add rounds to bf16 as the eager bf16 model does;
// id -1 contributes an exact zero row (ScaledEmbedding, :505-517).
// nn.Embedding raises on ids outside the table; here such an id (anything but the zero token -1 below 0, or >= rows)
// yields a NaN row and sets error bit 1.
__global__ void embed_sum_kernel(const long long* __restrict__ seq, int seq_stride, const bf16* __restrict__ wte,
                                 const bf16* const* __restrict__ tables, int n_q, int E, bf16* __restrict__ x,
                                 long long wte_rows, long long table_rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const long long* ids = seq + (long long)b * seq_stride;
  bool bad = ids[0] < -1 || ids[0] >= wte_rows;
  for (int cb = 0; cb < n_q; ++cb) bad |= ids[cb + 1] < -1 || ids[cb + 1] >= table_rows;
  if (bad && threadIdx.x == 0) atomicOr(&g_lm_dev_err, 1u);
  for (int d = threadIdx.x; d < E; d += blockDim.x) {
    float acc = 0.f;
    if (bad) {
      acc = __int_as_float(0x7fc00000);
    } else {
      for (int cb = 0; cb < n_q; ++cb) {
        const long long id = ids[cb + 1];
        const float e = id < 0 ? 0.f : b2f(tables[cb][id * E + d]);
        acc = cb == 0 ? e : b2f(f2b(acc + e));
      }
      const long long tid = ids[0];
      acc = b2f(f2b(acc + (tid < 0 ? 0.f : b2f(wte[tid * E + d]))));
    }
    x[(long long)b * E + d] = f2b(acc);
  }
}

// out[b] = table[id[b]] (zero row for id < 0): depth-transformer token embeddings (llama_streaming.py:738-742)
__global__ void embed_rows_kernel(const long long* __restrict__ ids, int id_stride, const bf16* __restrict__ table, int D,
                                  bf16* __restrict__ out, long long rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x;
  const long long id = ids[(long long)b * id_stride];
  const bool bad = id < -1 || id >= rows;
  if (bad && threadIdx.x == 0) atomicOr(&g_lm_dev_err, 1u);
  for (int d = threadIdx.x; d < D; d += blockDim.x)
    out[(long long)b * D + d] = bad ? f2b(__int_as_float(0x7fc00000)) : (id < 0 ? f2b(0.f) : table[id * D + d]);
}

// ---------------------------------------------------------------- RMSNorm, fp32 inside (lit_model.py:707-714;
// kyutai variant modules/transformer.py:34-48: var = eps + mean(x^2); y = x * (alpha * rsqrt(var)))
__global__ void rms_norm_kernel(const bf16* __restrict__ x, const bf16* __restrict__ w, bf16* __restrict__ y, int dim, float eps,
                                int kyutai) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[32];
  const int b = blockIdx.x;
  const bf16* xr = x + (long long)b * dim;
  float s = 0.f;
  for (int i = threadIdx.x; i < dim; i += blockDim.x) { const float v = b2f(xr[i]); s = fmaf(v, v, s); }
  s = warp_sum(s);
  if (threadIdx.x % 32 == 0) red[threadIdx.x / 32] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < blockDim.x / 32 ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  const float mean = red[0] / (float)dim;
  const float r = kyutai ? rsqrtf(eps + mean) : rsqrtf(mean + eps);
  for (int i = threadIdx.x; i < dim; i += blockDim.x) {
    const float v = b2f(xr[i]);
    const float o = kyutai ? v * (b2f(w[i]) * r) : (v * r) * b2f(w[i]);
    y[(long long)b * dim + i] = f2b(o);
  }
}

// ---------------------------------------------------------------- RoPE (rotate-half, bf16 cos/sin rows) + KV ring append
// Rows are (time, stream) pairs, time-major: row r = tl * B + b holds stream b at position *offset + tl (a decode step is
// tl == 0 for every row; a prefill chunk carries several consecutive positions per stream).
// qkv [row][n_kv][q_per_kv + 2][hs] (litgpt per-group interleave, llama_streaming.py:952-963; MHA is q_per_kv == 1);
// writes rotated q to q_out [row][n_head*hs] (head h = g*q_per_kv + j), rotated k and v into kv[2][B][n_kv][cap][hs] at
// slot (pos % cap)  (lit_model.py:560-573, 620-634).  Only the first rope_n dims rotate (rotary_percentage < 1,
// llama_streaming.py:979-982); the tables are [rope_rows][rope_n].  A position beyond the tables (the reference's
// cos.index_select would raise) poisons q/k with NaN and sets error bit 2.
__global__ void rope_kv_append_bf16_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ cosb, const bf16* __restrict__ sinb,
                                           const long long* __restrict__ offset, bf16* __restrict__ q_out, bf16* __restrict__ kv,
                                           int ostride, int B, int n_kv, int q_per_kv, int hs, int cap, int rope_n,
                                           long long rope_rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x / n_kv, g = blockIdx.x % n_kv;
  const int b = row % B;
  const long long pos = offset[(long long)b * ostride] + row / B;   // per-stream counters (ostride 1) or one shared (0)
  const int slot = (int)(pos % cap);
  const bool bad = pos >= rope_rows;
  if (bad && threadIdx.x == 0) atomicOr(&g_lm_dev_err, 2u);
  const bf16* base = qkv + ((long long)row * n_kv + g) * (q_per_kv + 2) * hs;
  const bf16* c = cosb + (bad ? 0 : pos) * rope_n;
  const bf16* s = sinb + (bad ? 0 : pos) * rope_n;
  bf16* kdst = kv + (((long long)b * n_kv + g) * cap + slot) * hs;
  bf16* vdst = kv + (long long)B * n_kv * cap * hs + (((long long)b * n_kv + g) * cap + slot) * hs;
  const int half = rope_n / 2;
  const bf16 nan = f2b(__int_as_float(0x7fc00000));
  for (int i = threadIdx.x; i < (q_per_kv + 1) * hs; i += blockDim.x) {
    const int j = i / hs, d = i % hs;           // j < q_per_kv: query j of the group; j == q_per_kv: the key
    const bf16* x = base + (long long)j * hs;
    bf16 o;
    if (d < rope_n) {
      // roped = (x * cos) + (rotated * sin), each op rounded to bf16 as the eager bf16 model does
      const float cd = b2f(c[d]), sd = b2f(s[d]);
      const float xv = b2f(x[d]);
      const float xr = d < half ? -b2f(x[d + half]) : b2f(x[d - half]);
      o = bad ? nan : f2b(b2f(f2b(xv * cd)) + b2f(f2b(xr * sd)));
    } else {
      o = x[d];
    }
    if (j < q_per_kv) q_out[((long long)row * n_kv * q_per_kv + (long long)g * q_per_kv + j) * hs + d] = o;
    else kdst[d] = o;
  }
  const bf16* vsrc = base + (long long)(q_per_kv + 1) * hs;
  for (int d = threadIdx.x; d < hs; d += blockDim.x) vdst[d] = vsrc[d];
}

// ---------------------------------------------------------------- Kyutai pair-RoPE (bf16 model) + KV ring append
// The Moshi-style LMModel's temporal transformer (models/model.py:364-389 over modules/transformer.py:375-419):
// qkv [row][3][H][hd] ((p h d) layout, transformer.py:391-393); (even, odd) pairs of q and k rotate by
// freqs[d/2] * (offset + tl) with everything in fp32 and ONE rounding to bf16 at the end (modules/rope.py:36-66);
// rotated q -> q_out [row][H*hd], rotated k and v -> kv[2][B][H][cap][hd] at slot pos % cap.
__global__ void rope_pair_kv_append_bf16_kernel(const bf16* __restrict__ qkv, const long long* __restrict__ offset, int ostride,
                                                bf16* __restrict__ q_out, bf16* __restrict__ kv, int B, int H, int hd, int cap,
                                                const float* __restrict__ freqs) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x / H, h = blockIdx.x % H;
  const int b = row % B;
  const long long off = offset[(long long)b * ostride];
  const long long pos = off + row / B;
  const int slot = (int)(pos % cap);
  const int HD = H * hd;
  const bf16* q = qkv + (long long)row * 3 * HD + h * hd;
  const bf16* k = q + HD;
  const bf16* v = q + 2 * HD;
  bf16* kdst = kv + (((long long)b * H + h) * cap + slot) * hd;
  bf16* vdst = kv + (long long)B * H * cap * hd + (((long long)b * H + h) * cap + slot) * hd;
  const float ts = __fadd_rn((float)off, (float)(row / B));     // offset.float() + arange(T) in fp32 (rope.py:37)
  for (int pr = threadIdx.x; pr < hd / 2; pr += blockDim.x) {
    const float ang = __fmul_rn(freqs[pr], ts);     // freqs = exp(ds * (-ln(max_period) * 2 / hd)) from the host (rope.py:35-36)
    const float c = cosf(ang), s = sinf(ang);
    const float qr = b2f(q[2 * pr]), qi = b2f(q[2 * pr + 1]);
    const float kr = b2f(k[2 * pr]), ki = b2f(k[2 * pr + 1]);
    bf16* qo = q_out + (long long)row * HD + h * hd;
    qo[2 * pr] = f2b(__fsub_rn(__fmul_rn(qr, c), __fmul_rn(qi, s)));
    qo[2 * pr + 1] = f2b(__fadd_rn(__fmul_rn(qr, s), __fmul_rn(qi, c)));
    kdst[2 * pr] = f2b(__fsub_rn(__fmul_rn(kr, c), __fmul_rn(ki, s)));
    kdst[2 * pr + 1] = f2b(__fadd_rn(__fmul_rn(kr, s), __fmul_rn(ki, c)));
    vdst[2 * pr] = v[2 * pr];
    vdst[2 * pr + 1] = v[2 * pr + 1];
  }
}

// ---------------------------------------------------------------- ring decode attention (one query position per row)
// one CTA per (G query heads sharing a kv head, row); 8 lanes share a key row (16 dims = 32 bytes each, so a warp load
// covers 4 whole 256-byte rows = 1 KB contiguous); per-group online softmax, combined across groups / warps at the end.
// Mask = RingKVCache.complete + (pos_k>=0)&(delta>=0)&(delta<context) (llama_streaming.py:983-992).
// Row r = tl*B + b queries stream b at position *offset + tl; all positions of the launch are already in the ring
// (the caller guarantees no slot a query still needs has been overwritten: see GPT.forward_global's prefill path).
// NS > 1 (key-split form): the work items are (row, head group, key chunk) triples walked by persistent CTAs
// (item = blockIdx.x + i * gridDim.x), so the 2048 equal (stream, head) jobs of the 7B step no longer run as 4.6 waves of 444
// resident CTAs (8 % of the kernel was an under-filled last wave) but as 13.8 rounds of thirds.  A chunk's unnormalised
// (max, sum, acc[HS]) goes to `ws`; the CTA that completes a (row, head group) -- found with one atomic counter, reset for
// the next launch -- combines the NS partials in chunk order, so the result does not depend on which CTA came last.
// ST > 0: the K/V rows travel through a per-lane cp.async ring in shared memory, ST - 1 sweeps (of 32 keys per CTA) in
// flight per warp instead of the one a register double buffer affords -- every lane copies and reads back only its own
// 16-byte pieces, so cp.async.wait_group is the only synchronisation.
template <int HS, int G, int NS, int ST>
__global__ void __launch_bounds__(256, (G == 1 ? 3 : 2)) ring_decode_attention_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kv,
                                                                    const long long* __restrict__ offset, bf16* __restrict__ out,
                                                                    int ostride, int B, int nh, int n_kv, int cap, int context,
                                                                    float scale, int rows, float* __restrict__ ws, int* __restrict__ arrive) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int DPL = HS / 8;  // dims per lane
  constexpr int PW = HS + 2;   // floats per partial: acc[HS], max, sum
  __shared__ float sm_m[G][8], sm_l[G][8], sm_acc[G][8][HS];
  __shared__ int sm_last;
  const int nhg = nh / G;
  const int n_items = rows * nhg * NS;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
  const int split = item % NS, hg = (item / NS) % nhg, row = item / (NS * nhg);
  const int h0 = hg * G;
  const int b = row % B;
  const int g = h0 / (nh / n_kv);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int grp = lane / 8, sub = lane % 8;
  const int nwarps = blockDim.x / 32;
  const long long pos = offset[(long long)b * ostride] + row / B;  // position of the query; its key/value were appended just before
  long long lo = pos - context + 1;
  if (lo < 0) lo = 0;
  if (lo < pos + 2 - cap) lo = pos + 2 - cap;  // ring quirk: the oldest slot is labelled end_offset and masked
  const long long nkeys_all = pos - lo + 1;
  const long long csz = NS == 1 ? nkeys_all : ((nkeys_all + NS - 1) / NS + 31) / 32 * 32;   // keys per chunk (whole 32-key sweeps)
  lo += (long long)split * csz;
  long long nkeys = nkeys_all - (long long)split * csz;
  if (nkeys > csz) nkeys = csz;
  if (nkeys < 0) nkeys = 0;
  const bf16* Kb = kv + ((long long)b * n_kv + g) * cap * HS;
  const bf16* Vb = Kb + (long long)B * n_kv * cap * HS;
  float qf[G][DPL];
#pragma unroll
  for (int u = 0; u < G; ++u) {
    // lane `sub` owns dims {p * 64 + sub * 8 + e}: piece p of all 8 lanes is one contiguous 128-byte run of a K/V row, so
    // every load instruction asks for whole 32-byte sectors (cp.async.cg bypasses L1 and would otherwise fetch each twice)
    const bf16* qp = q + ((long long)row * nh + h0 + u) * HS + sub * 8;
#pragma unroll
    for (int i = 0; i < DPL; ++i) qf[u][i] = b2f(qp[(i / 8) * 64 + i % 8]);
  }
  float m[G], l[G], acc[G][DPL];
#pragma unroll
  for (int u = 0; u < G; ++u) {
    m[u] = -INFINITY; l[u] = 0.f;
#pragma unroll
    for (int i = 0; i < DPL; ++i) acc[u][i] = 0.f;
  }
  // software pipeline: the K/V rows of the next iteration(s) are in flight while this one is reduced
  constexpr int CH = DPL / 8;          // 16-byte pieces of a K (or V) row per lane
  uint4 kr[CH], vr[CH], kn[ST > 0 ? 1 : CH], vn[ST > 0 ? 1 : CH];
  extern __shared__ __align__(16) unsigned char attn_ring[];
  uint4* ring = reinterpret_cast<uint4*>(attn_ring) + (ST > 0 ? warp * (ST * 2 * CH * 32) : 0);   // [stage][K pieces, V pieces][lane]
  auto issue_rows = [&](long long j0, int s) {
    const long long j = j0 + grp;
    const int slot = (int)((lo + (j < nkeys ? j : 0)) % cap);
    const uint4* kp = reinterpret_cast<const uint4*>(Kb + (long long)slot * HS) + sub;
    const uint4* vp = reinterpret_cast<const uint4*>(Vb + (long long)slot * HS) + sub;
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      cp_async16(&ring[(s * 2 * CH + i) * 32 + lane], kp + i * 8, 16);
      cp_async16(&ring[(s * 2 * CH + CH + i) * 32 + lane], vp + i * 8, 16);
    }
  };
  auto load_rows = [&](long long j0, uint4* kd, uint4* vd) {
    const long long j = j0 + grp;
    const int slot = (int)((lo + (j < nkeys ? j : 0)) % cap);
    const uint4* kp = reinterpret_cast<const uint4*>(Kb + (long long)slot * HS) + sub;
    const uint4* vp = reinterpret_cast<const uint4*>(Vb + (long long)slot * HS) + sub;
#pragma unroll
    for (int i = 0; i < DPL / 8; ++i) { kd[i] = __ldg(kp + i * 8); vd[i] = __ldg(vp + i * 8); }
  };
  const long long jstep = (long long)nwarps * 4;
  long long j0 = (long long)warp * 4;
  int stage = 0;
  if constexpr (ST > 0) {
#pragma unroll
    for (int s = 0; s < ST - 1; ++s) {
      if (j0 + s * jstep < nkeys) issue_rows(j0 + s * jstep, s);
      cp_async_commit();
    }
  } else {
    if (j0 < nkeys) load_rows(j0, kr, vr);
  }
  for (; j0 < nkeys; j0 += jstep) {
    const bool more = j0 + jstep < nkeys;
    if constexpr (ST > 0) {
      const int sn = stage == 0 ? ST - 1 : stage - 1;       // the stage consumed in the previous iteration
      if (j0 + (ST - 1) * jstep < nkeys) issue_rows(j0 + (ST - 1) * jstep, sn);
      cp_async_commit();
      cp_async_wait<ST - 1>();
#pragma unroll
      for (int i = 0; i < CH; ++i) {
        kr[i] = ring[(stage * 2 * CH + i) * 32 + lane];
        vr[i] = ring[(stage * 2 * CH + CH + i) * 32 + lane];
      }
      stage = stage + 1 == ST ? 0 : stage + 1;
    } else {
      if (more) load_rows(j0 + jstep, kn, vn);
    }
    const bool valid = j0 + grp < nkeys;
    float dot[G];
#pragma unroll
    for (int u = 0; u < G; ++u) dot[u] = 0.f;
#pragma unroll
    for (int i = 0; i < DPL / 8; ++i) {
      const bf16* kk = reinterpret_cast<const bf16*>(&kr[i]);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float kf = b2f(kk[e]);
#pragma unroll
        for (int u = 0; u < G; ++u) dot[u] = fmaf(qf[u][i * 8 + e], kf, dot[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < G; ++u) {
      dot[u] += __shfl_xor_sync(0xffffffffu, dot[u], 1);
      dot[u] += __shfl_xor_sync(0xffffffffu, dot[u], 2);
      dot[u] += __shfl_xor_sync(0xffffffffu, dot[u], 4);
    }
    if (valid) {
#pragma unroll
      for (int u = 0; u < G; ++u) {
        const float s = dot[u] * scale;
        const float m_new = fmaxf(m[u], s);
        const float corr = __expf(m[u] - m_new), pj = __expf(s - m_new);
        l[u] = l[u] * corr + pj;
#pragma unroll
        for (int i = 0; i < DPL / 8; ++i) {
          const bf16* vv = reinterpret_cast<const bf16*>(&vr[i]);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[u][i * 8 + e] = fmaf(pj, b2f(vv[e]), acc[u][i * 8 + e] * corr);
        }
        m[u] = m_new;
      }
    }
    if constexpr (ST == 0) {
      if (more) {
#pragma unroll
        for (int i = 0; i < DPL / 8; ++i) { kr[i] = kn[i]; vr[i] = vn[i]; }
      }
    }
  }
  if constexpr (ST > 0) cp_async_wait<0>();
#pragma unroll
  for (int u = 0; u < G; ++u) {
    // combine the 4 key groups of the warp (lanes sub, sub+8, sub+16, sub+24 hold the same dims)
    float mu = m[u], lu = l[u];
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {
      const float mo = __shfl_xor_sync(0xffffffffu, mu, o), lo_ = __shfl_xor_sync(0xffffffffu, lu, o);
      const float mn = fmaxf(mu, mo);
      const float ca = mn == -INFINITY ? 0.f : __expf(mu - mn), cb = mn == -INFINITY ? 0.f : __expf(mo - mn);
      lu = lu * ca + lo_ * cb;
#pragma unroll
      for (int i = 0; i < DPL; ++i) acc[u][i] = acc[u][i] * ca + __shfl_xor_sync(0xffffffffu, acc[u][i], o) * cb;
      mu = mn;
    }
    if (grp == 0) {
      if (sub == 0) { sm_m[u][warp] = mu; sm_l[u][warp] = lu; }
#pragma unroll
      for (int i = 0; i < DPL; ++i) sm_acc[u][warp][(i / 8) * 64 + sub * 8 + i % 8] = acc[u][i];
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < G * HS; idx += blockDim.x) {
    const int u = idx / HS, d = idx % HS;
    float mm = -INFINITY;
    for (int w = 0; w < nwarps; ++w) mm = fmaxf(mm, sm_m[u][w]);
    float ll = 0.f, a = 0.f;
    for (int w = 0; w < nwarps; ++w) {
      const float c = sm_m[u][w] == -INFINITY ? 0.f : __expf(sm_m[u][w] - mm);
      ll += sm_l[u][w] * c;
      a += sm_acc[u][w][d] * c;
    }
    if (NS == 1) {
      out[((long long)row * nh + h0 + u) * HS + d] = f2b(a / ll);
    } else {
      float* pw = ws + ((long long)item * G + u) * PW;
      pw[d] = a;
      if (d == 0) { pw[HS] = mm; pw[HS + 1] = ll; }
    }
  }
  if (NS > 1) {
    __threadfence();                 // this chunk's partial is visible before the arrival is counted
    __syncthreads();
    if (threadIdx.x == 0) {
      const int old = atomicAdd(&arrive[row * nhg + hg], 1);
      sm_last = old == NS - 1;
      if (sm_last) arrive[row * nhg + hg] = 0;      // ready for the next launch (all NS arrivals of this one are in)
    }
    __syncthreads();
    if (sm_last) {
      __threadfence();
      const long long first = ((long long)(row * nhg + hg) * NS) * G;   // the NS partials of this (row, head group) are adjacent items
      for (int idx = threadIdx.x; idx < G * HS; idx += blockDim.x) {
        const int u = idx / HS, d = idx % HS;
        float mm = -INFINITY;
#pragma unroll
        for (int sp = 0; sp < NS; ++sp) mm = fmaxf(mm, __ldcg(ws + (first + (long long)sp * G + u) * PW + HS));
        float ll = 0.f, a = 0.f;
#pragma unroll
        for (int sp = 0; sp < NS; ++sp) {
          const float* pw = ws + (first + (long long)sp * G + u) * PW;
          const float ms = __ldcg(pw + HS);
          const float c = ms == -INFINITY ? 0.f : __expf(ms - mm);
          ll += __ldcg(pw + HS + 1) * c;
          a += __ldcg(pw + d) * c;
        }
        out[((long long)row * nh + h0 + u) * HS + d] = f2b(a / ll);
      }
    }
  }
  __syncthreads();                   // the shared combine buffers are reused by the next item
  }
}

// ---------------------------------------------------------------- SiLU gating: out = silu(a) * b  (bf16 roundings as eager)
// ab [M][2*I] with a = cols [0,I), b = cols [I,2I) (fused fc_1|fc_2, or gating's view(B,T,2,-1), gating.py:16-19)
__global__ void silu_mul_kernel(const bf16* __restrict__ ab, bf16* __restrict__ out, int M, int I) {
  pdl_launch_dependents();
  pdl_wait();
  const long long total = (long long)M * I;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / I, c = i % I;
    const float a = b2f(ab[m * 2 * I + c]), b = b2f(ab[m * 2 * I + I + c]);
    const float s = b2f(f2b(a / (1.0f + expf(-a))));
    out[i] = f2b(s * b);
  }
}

// ---------------------------------------------------------------- depth-transformer attention (<= 8 keys, no RoPE)
// qkv [B][3][H][hd] ((p h d) layout, transformer.py:391-393); kvd [2][B][H][cap][hd]; step k: append at slot k,
// attend keys 0..k (cap == dep_q so the ring never wraps inside a frame).  ring_quirk != 0: the streaming form
// (forward_codecformer); 0: the non-streaming form (forward_local: KVCacheResult.from_kv keeps every key).
__global__ void depth_attention_kernel(const bf16* __restrict__ qkv, bf16* __restrict__ kvd, bf16* __restrict__ out, int B, int H,
                                       int hd, int cap, int step, int ring_quirk) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int lane = threadIdx.x;
  const int HD = H * hd;
  const bf16* qp = qkv + (long long)b * 3 * HD + h * hd;
  bf16* Kb = kvd + (((long long)b * H + h) * cap) * hd;
  bf16* Vb = Kb + (long long)B * H * cap * hd;
  for (int d = lane; d < hd; d += 32) {
    Kb[(long long)step * hd + d] = qp[HD + d];
    Vb[(long long)step * hd + d] = qp[2 * HD + d];
  }
  __syncwarp();
  const float scale = rsqrtf((float)hd);
  float sc[8];
  float mx = -INFINITY;
  // RingKVCache.complete labels slot end_offset % capacity with position end_offset (modules/transformer.py:258-263),
  // so on the last codebook step (end_offset == capacity) key 0 is masked by `delta >= 0`.
  const int j_lo = (ring_quirk && step + 2 - cap > 0) ? step + 2 - cap : 0;
  for (int j = j_lo; j <= step; ++j) {
    float dot = 0.f;
    for (int d = lane; d < hd; d += 32) dot = fmaf(b2f(qp[d]), b2f(Kb[(long long)j * hd + d]), dot);
    dot = warp_sum(dot) * scale;
    sc[j] = dot;
    mx = fmaxf(mx, dot);
  }
  float l = 0.f;
  for (int j = j_lo; j <= step; ++j) { sc[j] = __expf(sc[j] - mx); l += sc[j]; }
  for (int d = lane; d < hd; d += 32) {
    float a = 0.f;
    for (int j = j_lo; j <= step; ++j) a = fmaf(sc[j], b2f(Vb[(long long)j * hd + d]), a);
    out[(long long)b * HD + h * hd + d] = f2b(a / l);
  }
}

#include "lm_sample.cuh"

__global__ void sample_kernel(const bf16* __restrict__ logits, int V, int n_valid, int top_k, float temp, uint32_t seed,
                              const long long* __restrict__ step_counter, long long* __restrict__ tokens, int tok_stride) {
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  const uint32_t stepc = step_counter ? (uint32_t)(*step_counter) : 0u;
  sample_row(logits + (long long)row * V, n_valid, top_k, temp, seed, stepc, row, tokens + (long long)row * tok_stride);
}

}  // namespace rstnet
using namespace rstnet;

extern "C" int rstnet_lm_embed_sum_bf16(const int64_t* seq, int32_t seq_stride, const void* wte, int64_t wte_rows,
                                        const void* const* tables_dev, int64_t table_rows, int32_t n_q, int32_t E, void* x,
                                        int32_t rows, rstnet_stream_t stream) {
  RSTNET_REQUIRE(seq && wte && tables_dev && x && rows > 0 && wte_rows > 0 && table_rows > 0, "lm_embed_sum: bad argument");
  launch_pdl(embed_sum_kernel, dim3(rows), dim3(256), 0, (cudaStream_t)stream, (const long long*)seq, seq_stride, (const bf16*)wte,
             (const bf16* const*)tables_dev, n_q, E, (bf16*)x, (long long)wte_rows, (long long)table_rows);
  count_launch();
  return check_launch("lm_embed_sum");
}

extern "C" int rstnet_lm_embed_rows_bf16(const int64_t* ids, int32_t id_stride, const void* table, int64_t table_rows, int32_t D,
                                         void* out, int32_t rows, rstnet_stream_t stream) {
  RSTNET_REQUIRE(ids && table && out && rows > 0 && table_rows > 0, "lm_embed_rows: bad argument");
  launch_pdl(embed_rows_kernel, dim3(rows), dim3(128), 0, (cudaStream_t)stream, (const long long*)ids, id_stride, (const bf16*)table, D,
             (bf16*)out, (long long)table_rows);
  count_launch();
  return check_launch("lm_embed_rows");
}

extern "C" int rstnet_lm_rms_norm_bf16(const void* x, const void* w, void* y, int32_t rows, int32_t dim, float eps, int32_t kyutai,
                                       rstnet_stream_t stream) {
  RSTNET_REQUIRE(x && w && y && rows > 0 && dim > 0, "lm_rms_norm: bad argument");
  launch_pdl(rms_norm_kernel, dim3(rows), dim3(256), 0, (cudaStream_t)stream, (const bf16*)x, (const bf16*)w, (bf16*)y, dim, eps, kyutai);
  count_launch();
  return check_launch("lm_rms_norm");
}

extern "C" int rstnet_lm_rope_kv_append_bf16(const void* qkv, const void* cos_tab, const void* sin_tab, int64_t rope_rows,
                                             int32_t rope_n, const int64_t* offset, int32_t offset_stride, void* q_out, void* kv,
                                             int32_t rows, int32_t B, int32_t n_head, int32_t n_kv, int32_t hs, int32_t cap,
                                             rstnet_stream_t stream) {
  RSTNET_REQUIRE(qkv && cos_tab && sin_tab && offset && q_out && kv, "lm_rope_kv_append: null pointer");
  RSTNET_REQUIRE(rows > 0 && B > 0 && rows % B == 0, "lm_rope_kv_append: rows (%d) must be a multiple of the stream count (%d)", rows, B);
  RSTNET_REQUIRE(n_kv > 0 && n_head % n_kv == 0, "lm_rope_kv_append: n_head (%d) must be a multiple of n_kv (%d)", n_head, n_kv);
  RSTNET_REQUIRE(rope_n >= 0 && rope_n <= hs && rope_n % 2 == 0 && rope_rows > 0, "lm_rope_kv_append: bad rope table (%d of %d dims)", rope_n, hs);
  launch_pdl(rope_kv_append_bf16_kernel, dim3(rows * n_kv), dim3(64), 0, (cudaStream_t)stream, (const bf16*)qkv, (const bf16*)cos_tab,
             (const bf16*)sin_tab, (const long long*)offset, (bf16*)q_out, (bf16*)kv, offset_stride ? 1 : 0, B, n_kv, n_head / n_kv, hs,
             cap, rope_n, (long long)rope_rows);
  count_launch();
  return check_launch("lm_rope_kv_append");
}

extern "C" int rstnet_lm_rope_pair_kv_append_bf16(const void* qkv, const int64_t* offset, int32_t offset_stride, void* q_out, void* kv,
                                                  int32_t rows, int32_t B, int32_t H, int32_t hd, int32_t cap, const float* freqs,
                                                  rstnet_stream_t stream) {
  RSTNET_REQUIRE(qkv && offset && q_out && kv && freqs, "lm_rope_pair_kv_append: null pointer");
  RSTNET_REQUIRE(rows > 0 && B > 0 && rows % B == 0 && H > 0 && hd > 0 && hd % 2 == 0 && cap > 0, "lm_rope_pair_kv_append: bad shape");
  launch_pdl(rope_pair_kv_append_bf16_kernel, dim3(rows * H), dim3(64), 0, (cudaStream_t)stream, (const bf16*)qkv,
             (const long long*)offset, offset_stride ? 1 : 0, (bf16*)q_out, (bf16*)kv, B, H, hd, cap, freqs);
  count_launch();
  return check_launch("lm_rope_pair_kv_append");
}

extern "C" int64_t rstnet_lm_attention_split_workspace(int32_t rows, int32_t n_head, int32_t hs) {
  // [rows * n_head] int32 arrival counters (zeroed by the caller once), then 3 partials of (hs + 2) floats per (row, head)
  return (int64_t)rows * n_head * 4 + (int64_t)rows * n_head * 3 * (hs + 2) * 4;
}

extern "C" int rstnet_lm_ring_decode_attention_bf16(const void* q, const void* kv, const int64_t* offset, int32_t offset_stride,
                                                    void* out, int32_t rows, int32_t B, int32_t n_head, int32_t n_kv, int32_t hs,
                                                    int32_t cap, int32_t context, void* split_ws, rstnet_stream_t stream) {
  RSTNET_REQUIRE(q && kv && offset && out, "lm_ring_decode_attention: null pointer");
  RSTNET_REQUIRE(hs == 128 || hs == 64, "lm_ring_decode_attention: head_size must be 64 or 128 (got %d)", hs);
  RSTNET_REQUIRE(rows > 0 && B > 0 && rows % B == 0, "lm_ring_decode_attention: rows (%d) must be a multiple of the stream count (%d)", rows, B);
  RSTNET_REQUIRE(n_kv > 0 && n_head % n_kv == 0, "lm_ring_decode_attention: n_head (%d) must be a multiple of n_kv (%d)", n_head, n_kv);
  const float scale = 1.0f / sqrtf((float)hs);
  const int q_per_kv = n_head / n_kv;
  const int G = q_per_kv % 2 == 0 ? 2 : 1;   // query heads per CTA sharing the K/V rows (the rest of a group hits L2)
  cudaStream_t st = (cudaStream_t)stream;
  const int sms = sm_count();
  const int n_jobs = rows * (n_head / G);
  int* arrive = (int*)split_ws;
  float* ws = split_ws ? (float*)((char*)split_ws + (size_t)rows * n_head * 4) : nullptr;
  // split the keys only when the jobs would leave a badly filled last wave of resident CTAs
  const int resident = sms * (G == 1 ? 3 : 2);
  // opt-in by passing split_ws (measured slower than one CTA per job at the 7B shapes, DESIGN.md): only when the jobs exceed one wave
  const bool split = split_ws != nullptr && n_jobs > resident;
  static const int ring_stages = []() { const char* e = getenv("RSTNET_ATTN_STAGES"); return e ? atoi(e) : 4; }();   // 0: register double buffer
  const bool ring = ring_stages == 4 && !split;
  const int ring_bytes = ring ? 4 * 8 * 32 * (hs / 64) * 2 * 16 : 0;   // stages x warps x lanes x (K, V pieces) x 16 B
#define RSTNET_ATTN(HS_, G_)                                                                                                       \
  do {                                                                                                                             \
    if (split)                                                                                                                     \
      launch_pdl(ring_decode_attention_kernel<HS_, G_, 3, 0>, dim3(resident), dim3(256), 0, st, (const bf16*)q, (const bf16*)kv,   \
                 (const long long*)offset, (bf16*)out, offset_stride ? 1 : 0, B, n_head, n_kv, cap, context, scale, rows, ws, arrive); \
    else if (ring) {                                                                                                               \
      static unsigned long long attr = 0;                                                                                          \
      smem_optin(ring_decode_attention_kernel<HS_, G_, 1, 4>, ring_bytes, attr);                                                   \
      launch_pdl(ring_decode_attention_kernel<HS_, G_, 1, 4>, dim3(n_jobs), dim3(256), ring_bytes, st, (const bf16*)q,             \
                 (const bf16*)kv, (const long long*)offset, (bf16*)out, offset_stride ? 1 : 0, B, n_head, n_kv, cap, context,      \
                 scale, rows, (float*)nullptr, (int*)nullptr);                                                                     \
    } else                                                                                                                         \
      launch_pdl(ring_decode_attention_kernel<HS_, G_, 1, 0>, dim3(n_jobs), dim3(256), 0, st, (const bf16*)q, (const bf16*)kv,     \
                 (const long long*)offset, (bf16*)out, offset_stride ? 1 : 0, B, n_head, n_kv, cap, context, scale, rows,          \
                 (float*)nullptr, (int*)nullptr);                                                                                  \
  } while (0)
  if (hs == 128) { if (G == 2) RSTNET_ATTN(128, 2); else RSTNET_ATTN(128, 1); }
  else           { if (G == 2) RSTNET_ATTN(64, 2); else RSTNET_ATTN(64, 1); }
#undef RSTNET_ATTN
  count_launch();
  return check_launch("lm_ring_decode_attention");
}

extern "C" int rstnet_lm_silu_mul_bf16(const void* ab, void* out, int32_t M, int32_t I, rstnet_stream_t stream) {
  RSTNET_REQUIRE(ab && out && M > 0 && I > 0, "lm_silu_mul: bad argument");
  const long long total = (long long)M * I;
  int g = ceil_div(total, 256);
  if (g > sm_count() * 8) g = sm_count() * 8;
  launch_pdl(silu_mul_kernel, dim3(g), dim3(256), 0, (cudaStream_t)stream, (const bf16*)ab, (bf16*)out, M, I);
  count_launch();
  return check_launch("lm_silu_mul");
}

extern "C" int rstnet_lm_depth_attention_bf16(const void* qkv, void* kvd, void* out, int32_t B, int32_t H, int32_t hd, int32_t cap,
                                              int32_t step, int32_t ring_quirk, rstnet_stream_t stream) {
  RSTNET_REQUIRE(qkv && kvd && out, "lm_depth_attention: null pointer");
  RSTNET_REQUIRE(step >= 0 && step < cap && cap <= 8, "lm_depth_attention: step %d / capacity %d (<= 8) out of range", step, cap);
  launch_pdl(depth_attention_kernel, dim3(B * H), dim3(32), 0, (cudaStream_t)stream, (const bf16*)qkv, (bf16*)kvd, (bf16*)out, B, H, hd, cap,
             step, ring_quirk);
  count_launch();
  return check_launch("lm_depth_attention");
}

extern "C" int rstnet_lm_sample_bf16(const void* logits, int32_t rows, int32_t V, int32_t n_valid, int32_t top_k, float temp,
                                     uint32_t seed, const int64_t* step_counter, int64_t* tokens, int32_t tok_stride,
                                     rstnet_stream_t stream) {
  RSTNET_REQUIRE(logits && tokens && rows > 0 && V > 0, "lm_sample: bad argument");
  RSTNET_REQUIRE(top_k <= SAMPLE_CAND && (top_k == 0 || temp > 0.f), "lm_sample: top_k <= %d and temp > 0 required (top_k=%d)", SAMPLE_CAND, top_k);
  if (n_valid <= 0 || n_valid > V) n_valid = V;
  if (top_k > n_valid) top_k = n_valid;   // torch.topk would raise; the whole support is the natural reading
  launch_pdl(sample_kernel, dim3(rows), dim3(1024), 0, (cudaStream_t)stream, (const bf16*)logits, V, n_valid, top_k, temp, (uint32_t)seed,
             (const long long*)step_counter, (long long*)tokens, tok_stride);
  count_launch();
  return check_launch("lm_sample");
}
