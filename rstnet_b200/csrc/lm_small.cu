// HBM-bound bf16 kernels of the speech-text LM decode step: embedding sum, RMSNorm (two variants),
// rotate-half RoPE + ring-KV append, ring decode attention, SiLU gating, depth-transformer attention,
// embedding gather, greedy / top-k sampling.  One token per stream (T == 1): rows are streams.
#include <cuda_bf16.h>

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
// yields a NaN row and sets error bit 0 (1).
__global__ void embed_sum_kernel(const long long* __restrict__ seq, int seq_stride, const bf16* __restrict__ wte,
                                 const bf16* const* __restrict__ tables, int n_q, int E, bf16* __restrict__ x,
                                 long long wte_rows, long long table_rows) {
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
// cos.index_select would raise) poisons q/k with NaN and sets error bit 1 (2).
// Row map (ragged prefill of some streams): with row_stream set, row r is stream row_stream[r] at position
// offset[row_stream[r]] + row_tl[r] instead; row_stream[r] == -1 is a padding row that reads and writes nothing.  A runtime
// branch, not a second instantiation, so the uniform and the mapped launch run one compiled body (DESIGN.md §6).
// Page table (paged KV, GPT.streaming(B, kv_pages=N)): the logical ring is unchanged -- position p in slot p % cap -- but
// slot s of stream b lives in page page_table[b * pages_stride + (s >> log2_page)], row s & (2^log2_page - 1), of a pool
// kv[n_pages][2][n_kv][2^log2_page][hs].  A page entry of -1 is unmapped: a row whose own slot falls on one behaves like a
// padding row.  page_table == nullptr is the contiguous ring, again by a runtime branch of the same body.
__global__ void rope_kv_append_bf16_kernel(const bf16* __restrict__ qkv, const bf16* __restrict__ cosb, const bf16* __restrict__ sinb,
                                           const long long* __restrict__ offset, bf16* __restrict__ q_out, bf16* __restrict__ kv,
                                           int ostride, int B, int n_kv, int q_per_kv, int hs, int cap, int rope_n,
                                           long long rope_rows, const int* __restrict__ row_stream, const int* __restrict__ row_tl,
                                           const int* __restrict__ page_table, int pages_stride, int log2_page) {
  const int row = blockIdx.x / n_kv, g = blockIdx.x % n_kv;
  int b, tl;
  if (row_stream) {
    b = row_stream[row];
    if (b < 0) return;
    tl = row_tl[row];
  } else {
    b = row % B;
    tl = row / B;
  }
  const long long pos = offset[(long long)b * ostride] + tl;   // per-stream counters (ostride 1) or one shared (0)
  const int slot = (int)(pos % cap);
  bf16* kdst;
  long long vofs;   // V row of a slot = its K row + vofs
  if (page_table) {
    const int page = page_table[(long long)b * pages_stride + (slot >> log2_page)];
    if (page < 0) return;   // unmapped: nothing read, nothing written
    kdst = kv + ((((long long)page * 2 * n_kv + g) << log2_page) + (slot & ((1 << log2_page) - 1))) * hs;
    vofs = ((long long)n_kv << log2_page) * hs;
  } else {
    kdst = kv + (((long long)b * n_kv + g) * cap + slot) * hs;
    vofs = (long long)B * n_kv * cap * hs;
  }
  bf16* vdst = kdst + vofs;
  const bool bad = pos >= rope_rows;
  if (bad && threadIdx.x == 0) atomicOr(&g_lm_dev_err, 2u);
  const bf16* base = qkv + ((long long)row * n_kv + g) * (q_per_kv + 2) * hs;
  const bf16* c = cosb + (bad ? 0 : pos) * rope_n;
  const bf16* s = sinb + (bad ? 0 : pos) * rope_n;
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
// Page table (paged KV, LMModel.streaming(B, kv_pages=N)): as rope_kv_append_bf16_kernel's -- slot s of stream b lives in
// page page_table[b * pages_stride + (s >> log2_page)], row s & (2^log2_page - 1), of a pool kv[n_pages][2][H][2^log2_page][hd],
// and a row whose own slot falls on an unmapped page (-1) writes nothing, q_out included.  A runtime branch of the same body.
// Row map (ragged chunks of many streams, LMModel.forward / moshi.score_many): as rope_kv_append_bf16_kernel's -- row r is
// stream row_stream[r] at position offset[row_stream[r]] + row_tl[r], and row_stream[r] == -1 is a padding row that reads
// and writes nothing, q_out included.  The angle is fp32(offset) + fp32(tl) either way.  Again a runtime branch.
__global__ void rope_pair_kv_append_bf16_kernel(const bf16* __restrict__ qkv, const long long* __restrict__ offset, int ostride,
                                                bf16* __restrict__ q_out, bf16* __restrict__ kv, int B, int H, int hd, int cap,
                                                const float* __restrict__ freqs, const int* __restrict__ page_table,
                                                int pages_stride, int log2_page, const int* __restrict__ row_stream,
                                                const int* __restrict__ row_tl) {
  const int row = blockIdx.x / H, h = blockIdx.x % H;
  int b, tl;
  if (row_stream) {
    b = row_stream[row];
    if (b < 0) return;
    tl = row_tl[row];
  } else {
    b = row % B;
    tl = row / B;
  }
  const long long off = offset[(long long)b * ostride];
  const long long pos = off + tl;
  const int slot = (int)(pos % cap);
  const int HD = H * hd;
  const bf16* q = qkv + (long long)row * 3 * HD + h * hd;
  const bf16* k = q + HD;
  const bf16* v = q + 2 * HD;
  bf16* kdst;
  long long vofs;   // V row of a slot = its K row + vofs
  if (page_table) {
    const int page = page_table[(long long)b * pages_stride + (slot >> log2_page)];
    if (page < 0) return;   // unmapped: nothing read, nothing written
    kdst = kv + ((((long long)page * 2 * H + h) << log2_page) + (slot & ((1 << log2_page) - 1))) * hd;
    vofs = ((long long)H << log2_page) * hd;
  } else {
    kdst = kv + (((long long)b * H + h) * cap + slot) * hd;
    vofs = (long long)B * H * cap * hd;
  }
  bf16* vdst = kdst + vofs;
  const float ts = __fadd_rn((float)off, (float)tl);     // offset.float() + arange(T) in fp32 (rope.py:37)
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
// Row r = tl*B + b queries stream b at position *offset + tl, or, with row_stream set, the row map of
// rope_kv_append_bf16_kernel (padding rows write nothing); all positions of the launch are already in the ring
// (the caller guarantees no slot a query still needs has been overwritten: see GPT.forward_global's prefill path).
// The K/V rows travel through a per-lane cp.async ring in shared memory, ATT_STAGES - 1 sweeps (of 32 keys per CTA) in
// flight per warp -- every lane copies and reads back only its own 16-byte pieces, so cp.async.wait_group is the only
// synchronisation.
// Page table: slot addressing of rope_kv_append_bf16_kernel.  A row whose own slot is on an unmapped page writes zeros; a
// key slot on an unmapped page is never read (its cp.async copies 0 bytes and fills zeros) -- callers keep every key of a
// window mapped (GPT.streaming's host guard), so that never enters a real result.  Keys are visited in the same order
// and summed in the same order as in the contiguous ring: only the addresses differ.
constexpr int ATT_STAGES = 4;
constexpr int ATT_WARPS = 8;
template <int HS, int G>
__global__ void __launch_bounds__(ATT_WARPS * 32, (G == 1 ? 3 : 2)) ring_decode_attention_kernel(const bf16* __restrict__ q, const bf16* __restrict__ kv,
                                                                    const long long* __restrict__ offset, bf16* __restrict__ out,
                                                                    int ostride, int B, int nh, int n_kv, int cap, int context,
                                                                    float scale, const int* __restrict__ row_stream,
                                                                    const int* __restrict__ row_tl, const int* __restrict__ page_table,
                                                                    int pages_stride, int log2_page) {
  constexpr int ST = ATT_STAGES;
  constexpr int DPL = HS / 8;  // dims per lane
  __shared__ float sm_m[G][ATT_WARPS], sm_l[G][ATT_WARPS], sm_acc[G][ATT_WARPS][HS];
  const int nhg = nh / G;
  const int hg = blockIdx.x % nhg, row = blockIdx.x / nhg;
  const int h0 = hg * G;
  int b, tl;
  if (row_stream) {
    b = row_stream[row];
    if (b < 0) return;   // the whole CTA serves this row
    tl = row_tl[row];
  } else {
    b = row % B;
    tl = row / B;
  }
  const int g = h0 / (nh / n_kv);
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int grp = lane / 8, sub = lane % 8;
  constexpr int nwarps = ATT_WARPS;
  const long long pos = offset[(long long)b * ostride] + tl;  // position of the query; its key/value were appended just before
  long long lo = pos - context + 1;
  if (lo < 0) lo = 0;
  if (lo < pos + 2 - cap) lo = pos + 2 - cap;  // ring quirk: the oldest slot is labelled end_offset and masked
  const long long nkeys = pos - lo + 1;
  // K row of slot s: Kb + r(s) * HS with r(s) = s (contiguous) or page(s) * page_rows + (s & pmask); V row = K row + vofs
  const int* pt = nullptr;
  const bf16* Kb;
  long long vofs, page_rows = 0;
  const int pmask = (1 << log2_page) - 1;
  if (page_table) {
    pt = page_table + (long long)b * pages_stride;
    if (pt[(int)(pos % cap) >> log2_page] < 0) {   // the query's own position is unmapped: a finite, all-zero output
      for (int idx = threadIdx.x; idx < G * HS; idx += blockDim.x) out[((long long)row * nh + h0) * HS + idx] = f2b(0.f);
      return;
    }
    Kb = kv + ((long long)g << log2_page) * HS;
    vofs = ((long long)n_kv << log2_page) * HS;
    page_rows = (2LL * n_kv) << log2_page;
  } else {
    Kb = kv + ((long long)b * n_kv + g) * cap * HS;
    vofs = (long long)B * n_kv * cap * HS;
  }
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
  // software pipeline: the K/V rows of the next iterations are in flight while this one is reduced
  constexpr int CH = DPL / 8;          // 16-byte pieces of a K (or V) row per lane
  uint4 kr[CH], vr[CH];
  extern __shared__ __align__(16) unsigned char attn_ring[];
  uint4* ring = reinterpret_cast<uint4*>(attn_ring) + warp * (ST * 2 * CH * 32);   // [stage][K pieces, V pieces][lane]
  auto issue_rows = [&](long long j0, int s) {
    const long long j = j0 + grp;
    const int slot = (int)((lo + (j < nkeys ? j : 0)) % cap);
    long long r = slot;
    int bytes = 16;
    if (pt) {
      const int page = pt[slot >> log2_page];
      bytes = page < 0 ? 0 : 16;
      r = page < 0 ? 0 : page * page_rows + (slot & pmask);
    }
    const uint4* kp = reinterpret_cast<const uint4*>(Kb + r * HS) + sub;
    const uint4* vp = reinterpret_cast<const uint4*>(Kb + vofs + r * HS) + sub;
#pragma unroll
    for (int i = 0; i < CH; ++i) {
      cp_async16(&ring[(s * 2 * CH + i) * 32 + lane], kp + i * 8, bytes);
      cp_async16(&ring[(s * 2 * CH + CH + i) * 32 + lane], vp + i * 8, bytes);
    }
  };
  const long long jstep = (long long)nwarps * 4;
  long long j0 = (long long)warp * 4;
  int stage = 0;
#pragma unroll
  for (int s = 0; s < ST - 1; ++s) {
    if (j0 + s * jstep < nkeys) issue_rows(j0 + s * jstep, s);
    cp_async_commit();
  }
  for (; j0 < nkeys; j0 += jstep) {
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
  }
  cp_async_wait<0>();
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
    out[((long long)row * nh + h0 + u) * HS + d] = f2b(a / ll);
  }
}

// one CTA per (row, head group); the dynamic shared memory is the cp.async ring: stages x warps x lanes x (K, V pieces) x 16 B
template <int HS, int G>
void launch_ring_decode_attention(cudaStream_t st, const bf16* q, const bf16* kv, const long long* offset, bf16* out, int ostride,
                                  int rows, int B, int nh, int n_kv, int cap, int context, float scale, const int* row_stream,
                                  const int* row_tl, const int* page_table, int pages_stride, int log2_page) {
  constexpr int smem = ATT_STAGES * ATT_WARPS * 32 * (HS / 64) * 2 * 16;
  static unsigned long long attr = 0;
  smem_optin(ring_decode_attention_kernel<HS, G>, smem, attr);
  ring_decode_attention_kernel<HS, G><<<rows * (nh / G), ATT_WARPS * 32, smem, st>>>(q, kv, offset, out, ostride, B, nh, n_kv, cap, context, scale,
                                                                                                    row_stream, row_tl, page_table, pages_stride,
                                                                                                    log2_page);
}

// ---------------------------------------------------------------- SiLU gating: out = silu(a) * b  (bf16 roundings as eager)
// ab [M][2*I] with a = cols [0,I), b = cols [I,2I) (fused fc_1|fc_2, or gating's view(B,T,2,-1), gating.py:16-19)
__global__ void silu_mul_kernel(const bf16* __restrict__ ab, bf16* __restrict__ out, int M, int I) {
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

// ---------------------------------------------------------------- sampling (utils/sampling.py:85-154)
__device__ __forceinline__ uint32_t hash_u32(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  uint32_t h = a * 0x9E3779B1u ^ (b + 0x7F4A7C15u) * 0x85EBCA77u ^ (c + 0x165667B1u) * 0xC2B2AE3Du ^ (d * 0x27D4EB2Fu);
  h ^= h >> 16; h *= 0x7FEB352Du; h ^= h >> 15; h *= 0x846CA68Bu; h ^= h >> 16;
  return h;
}

// logits [rows][V] bf16, candidates restricted to ids < n_valid.  top_k <= 0: argmax (first maximum).
// top_k > 0: the top_k largest logits, weights exp((l - max)/temp), token = argmax_i w_i / Exp(1)_i
// (= torch's exponential-noise multinomial over the top-k probabilities, sampling.py:43-46, 57-59).
//
// Large vocabularies (the 152k text head) first shrink the row to a candidate list: bf16 has 16 key bits, so two
// 256-bin histogram passes give the exact key of the top_k-th largest logit; every logit with key >= that threshold
// (top_k of them plus ties) is compacted into shared memory and the ordered selection below runs on the list instead
// of re-scanning the row top_k times.  Same result as the full scan: (value desc, index asc) order.
constexpr int SAMPLE_CAND = 1024;
constexpr int SAMPLE_HISTS = 16;

// The one order key of every path: monotone in the bf16 value under float comparison, so -0 and +0 share a key (equal
// logits tie, and ties go lowest index first), and NaN takes key 0, below -inf (0x7F): no path counts a NaN id.
__device__ __forceinline__ uint32_t bf16_order_key(bf16 v) {
  uint32_t u = (uint32_t)__bfloat16_as_ushort(v);
  if ((u & 0x7FFFu) > 0x7F80u) return 0u;
  if (u == 0x8000u) u = 0u;
  return (u & 0x8000u) ? (~u & 0xFFFFu) : (u | 0x8000u);
}

// block-wide argmax in the order (value desc, index asc); every thread returns the winner
__device__ __forceinline__ void block_argmax(float& bv, int& bi, float* s_val, int* s_idx) {
  const int tid = threadIdx.x, nthr = blockDim.x;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
  }
  __syncthreads();   // the previous round's readers are done with s_val / s_idx
  if (tid % 32 == 0) { s_val[tid / 32] = bv; s_idx[tid / 32] = bi; }
  __syncthreads();
  if (tid < 32) {
    bv = tid < nthr / 32 ? s_val[tid] : -INFINITY;
    bi = tid < nthr / 32 ? s_idx[tid] : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (tid == 0) { s_val[0] = bv; s_idx[0] = bi; }
  }
  __syncthreads();
  bv = s_val[0];
  bi = s_idx[0];
}

__device__ __forceinline__ float gumbel_of(uint32_t seed, uint32_t stepc, uint32_t row, uint32_t id) {
  const uint32_t u = hash_u32(seed, stepc, row, id);
  const float uni = ((float)(u >> 8) + 0.5f) * (1.0f / 16777216.0f);  // (0,1)
  return -logf(-logf(uni));   // argmax_i (l_i/temp + G_i)  ==  argmax_i softmax(l/temp)_i / Exp(1)_i
}

// the multinomial score of id i: one expression shared by the multinomial, top_k > 64 and nucleus draws, so a token
// kept by two of them has the same score in both
__device__ __forceinline__ float multinomial_score(float l, float inv_t, uint32_t seed, uint32_t stepc, uint32_t row, uint32_t i) {
  return l * inv_t + gumbel_of(seed, stepc, row, i);
}

// Nucleus: bf16_order_key, and the weight exp((l - max) / temp) in 2^-40 fixed point (<= 2^40 per id, < 2^58 for
// 152 064 ids).  Integer sums give the same mass whatever the order of the atomics.  NaN logits and weights below 2^-40
// weigh 0.
constexpr int SAMPLE_MHISTS = 4;
__device__ __forceinline__ unsigned long long nucleus_weight(float l, float mx, float inv_t) {
  const float w = expf((l - mx) * inv_t);
  return w > 0.f ? (unsigned long long)(w * 1099511627776.0f) : 0ull;
}
__device__ __forceinline__ float key_value(uint32_t k) {   // inverse of bf16_order_key (key 0: a NaN)
  const unsigned short u = (k & 0x8000u) ? (unsigned short)(k & 0x7FFFu) : (unsigned short)(~k & 0xFFFFu);
  return b2f(__ushort_as_bfloat16(u));
}

// top_k == 0: argmax.  1..64: ordered selection of the top-k (below), noise keyed by rank.  65..SAMPLE_CAND: threshold
// select (the k largest by (value desc, index asc), found with the histogram + candidate list), noise keyed by token id.
// top_k < 0: multinomial over all n_valid ids (sample_token with top_k == 0, utils/sampling.py:97-101).
// top_k != 0 and 0 < top_p < 1: nucleus (sample_top_p, utils/sampling.py:66-82; it takes precedence over top_k as in
// sample_token).  With w_i = exp((l_i - max) / temp) and Z = sum of w over the ids < n_valid, id t is kept iff the mass of
// the ids before it in the order (logit desc, index asc) is <= top_p * Z, so the kept set is a prefix holding the top
// token.  Equal logits have equal weights; at the cut they are taken lowest index first.  The draw is the first maximum
// of the multinomial score over the kept ids, so it equals the top_k < 0 draw whenever that draw is kept (in particular
// whenever every id is kept).  The cut: two 256-bin passes over the order key with counts and fixed-point masses.
// Deviation: the reference's masked audio samplers (sample_token_audio[_2048] with top_p > 0) give NaN, because they mask
// with -inf before the cumulative sum; here the distribution is restricted to the ids < n_valid and renormalised.
//
// Order and edges, the same in every mode and on every path (full scan, candidate list, tie walk):
// - The order is (value desc, index asc) under float comparison: -0 and +0 are equal logits.
// - A NaN logit is never a candidate: it takes no top-k slot and is never drawn.  With fewer than top_k other ids, the
//   top-k keeps them all.
// - A +inf logit scores +inf wherever the score is l / temp + Gumbel noise (equal scores: the lowest id), as it wins the
//   argmax; top_k <= 64 weighs each +inf id 1 and every other id 0.
// - If no kept id scores above -inf (in particular when every id < n_valid is -inf or NaN), the draw is id 0.  So every
//   draw is an id in [0, n_valid).
// tests/sampler_restatement.py restates every draw on the host.
// All threads of the block call it (any block size that is a multiple of 32, <= 1024); writes *token_out.
__device__ __noinline__ void sample_row(const bf16* __restrict__ lr, int n_valid, int top_k, float temp, float top_p, uint32_t seed,
                                        uint32_t stepc, int row, long long* __restrict__ token_out) {
  __shared__ float s_val[32];
  __shared__ int s_idx[32];
  __shared__ float top_v[64];
  __shared__ int top_i[64];
  __shared__ int hist[SAMPLE_HISTS][256];
  __shared__ float cand_v[SAMPLE_CAND];
  __shared__ int cand_i[SAMPLE_CAND];
  __shared__ int s_sel[5];   // [0] high-byte bin, [1] count above the threshold key, [2] threshold key, [3] candidate count, [4] ties taken
  __shared__ unsigned long long mhist[SAMPLE_MHISTS][256];
  __shared__ unsigned long long s_mass[2];   // nucleus: [0] mass above the cut bin / key, [1] floor(top_p * Z)
  const int tid = threadIdx.x, nthr = blockDim.x;

  if (top_k != 0 && top_p > 0.f && top_p < 1.f) {
    const float inv_t = 1.0f / temp;
    float mx = -INFINITY;
    int mi = 0;
    for (int i = tid; i < n_valid; i += nthr) mx = fmaxf(mx, b2f(lr[i]));
    block_argmax(mx, mi, s_val, s_idx);
    if (mx > -INFINITY) {   // (no id above -inf: the top_k paths below, which draw id 0)
      int* myh = hist[(tid / 32) % SAMPLE_HISTS];
      unsigned long long* mym = mhist[(tid / 32) % SAMPLE_MHISTS];
      for (int pass = 0; pass < 2; ++pass) {
        for (int i = tid; i < SAMPLE_HISTS * 256; i += nthr) (&hist[0][0])[i] = 0;
        for (int i = tid; i < SAMPLE_MHISTS * 256; i += nthr) (&mhist[0][0])[i] = 0ull;
        __syncthreads();
        const uint32_t b1 = pass ? (uint32_t)s_sel[0] : 0u;
        // Warp-aggregated: the lanes of a warp that fall into one bin add their count and mass with one atomic each. An LM
        // head occupies a handful of high-byte bins, so one atomic per id would serialise on them.  The masses (< 2^41
        // per id) are summed across the lanes in two 20-bit halves, which cannot overflow 32 bits.
        for (int base = 0; base < n_valid; base += nthr) {
          const int i = base + tid;
          uint32_t bin = 0xFFFFFFFFu;   // no bin: past the row, or outside the bin of pass 1
          unsigned long long w = 0;
          if (i < n_valid) {
            const bf16 v = lr[i];
            const uint32_t k = bf16_order_key(v);
            if (k && (pass == 0 || (k >> 8) == b1)) {
              bin = pass ? (k & 255u) : (k >> 8);
              w = nucleus_weight(b2f(v), mx, inv_t);
            }
          }
          const unsigned peers = __match_any_sync(0xffffffffu, bin);
          const unsigned lo = __reduce_add_sync(peers, (unsigned)(w & 0xFFFFFull));
          const unsigned hi = __reduce_add_sync(peers, (unsigned)(w >> 20));
          if (bin != 0xFFFFFFFFu && (int)(tid % 32) == __ffs(peers) - 1) {
            atomicAdd(&myh[bin], __popc(peers));
            const unsigned long long m = ((unsigned long long)hi << 20) + lo;
            if (m) atomicAdd(&mym[bin], m);
          }
        }
        __syncthreads();
        if (tid < 256) {
          int c = 0;
          unsigned long long m = 0;
#pragma unroll
          for (int h = 0; h < SAMPLE_HISTS; ++h) c += hist[h][tid];
#pragma unroll
          for (int h = 0; h < SAMPLE_MHISTS; ++h) m += mhist[h][tid];
          hist[0][tid] = c;
          mhist[0][tid] = m;
        }
        __syncthreads();
        if (tid == 0) {
          unsigned long long above = 0;
          if (pass == 0) {
            for (int b = 0; b < 256; ++b) above += mhist[0][b];   // Z
            s_mass[1] = (unsigned long long)((double)top_p * (double)above);
            above = 0;
          } else {
            above = s_mass[0];
          }
          const unsigned long long cut_mass = s_mass[1];
          int cut = 0;
          unsigned long long cut_above = 0;
          // the lowest non-empty bin whose mass above is <= top_p * Z: every id above it is kept, none below it
          for (int b = 255; b >= 0; --b) {
            if (!hist[0][b]) continue;
            if (above > cut_mass) break;
            cut = b;
            cut_above = above;
            above += mhist[0][b];
          }
          s_mass[0] = cut_above;
          if (pass == 0) {
            s_sel[0] = cut;
          } else {
            const uint32_t key = ((uint32_t)s_sel[0] << 8) | (uint32_t)cut;
            const int cnt = hist[0][cut];
            const unsigned long long w = nucleus_weight(key_value(key), mx, inv_t);
            const unsigned long long fit = w ? (cut_mass - cut_above) / w + 1ull : (unsigned long long)cnt;
            s_sel[1] = fit < (unsigned long long)cnt ? (int)fit : cnt;   // ties at the cut key to keep, lowest ids first
            s_sel[2] = (int)key;
            s_sel[3] = cnt;
            s_sel[4] = 0x7fffffff;   // the largest kept id at the cut key
          }
        }
        __syncthreads();
      }
      const uint32_t thr = (uint32_t)s_sel[2];
      const int need = s_sel[1], cnt = s_sel[3];
      if (need < cnt) {
        if (cnt <= SAMPLE_CAND) {
          if (tid == 0) s_sel[0] = 0;
          __syncthreads();
          for (int i = tid; i < n_valid; i += nthr)
            if (bf16_order_key(lr[i]) == thr) cand_i[atomicAdd(&s_sel[0], 1)] = i;
          __syncthreads();
          for (int t = tid; t < cnt; t += nthr) {
            const int id = cand_i[t];
            int rank = 0;
            for (int j = 0; j < cnt; ++j) rank += cand_i[j] < id ? 1 : 0;
            if (rank == need - 1) s_sel[4] = id;
          }
        } else {
          // more than SAMPLE_CAND logits share the cut value: walk the row in index order, counting ties
          if (tid == 0) s_sel[0] = 0;
          for (int base = 0; base < n_valid; base += nthr) {
            const int i = base + tid;
            const bool tie = i < n_valid && bf16_order_key(lr[i]) == thr;
            const unsigned bal = __ballot_sync(0xffffffffu, tie);
            const int wpre = __popc(bal & ((1u << (tid % 32)) - 1u));
            __syncthreads();
            if (tid % 32 == 0) s_idx[tid / 32] = __popc(bal);
            __syncthreads();
            int before = s_sel[0];
            for (int w = 0; w < tid / 32; ++w) before += s_idx[w];
            if (tie && before + wpre == need - 1) s_sel[4] = i;
            __syncthreads();
            if (tid == 0) { int t = 0; for (int w = 0; w < nthr / 32; ++w) t += s_idx[w]; s_sel[0] += t; }
            __syncthreads();
            if (s_sel[0] >= need) break;
          }
        }
        __syncthreads();
      }
      const int last = s_sel[4];
      float bv = -INFINITY;
      int bi = 0x7fffffff;
      for (int i = tid; i < n_valid; i += nthr) {
        const bf16 v = lr[i];
        const uint32_t k = bf16_order_key(v);
        if (k > thr || (k == thr && i <= last)) {
          const float sc = multinomial_score(b2f(v), inv_t, seed, stepc, (uint32_t)row, (uint32_t)i);
          if (sc > bv) { bv = sc; bi = i; }
        }
      }
      block_argmax(bv, bi, s_val, s_idx);
      if (tid == 0) *token_out = bv > -INFINITY ? bi : 0;   // no kept id scores above -inf: id 0
      return;
    }
  }

  if (top_k < 0) {   // full multinomial
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    const float inv_t = 1.0f / temp;
    for (int i = tid; i < n_valid; i += nthr) {
      const float sc = multinomial_score(b2f(lr[i]), inv_t, seed, stepc, (uint32_t)row, (uint32_t)i);
      if (sc > bv) { bv = sc; bi = i; }
    }
    block_argmax(bv, bi, s_val, s_idx);
    if (tid == 0) *token_out = bv > -INFINITY ? bi : 0;
    return;
  }

  const bool big = top_k > 64;
  const int kk = top_k <= 0 ? 1 : (big ? top_k : top_k);
  int n_items = n_valid;
  bool from_list = false;
  if (big || (kk > 1 && n_valid > 4 * SAMPLE_CAND)) {
    int* myh = hist[(tid / 32) % SAMPLE_HISTS];
    for (int pass = 0; pass < 2; ++pass) {
      for (int i = tid; i < SAMPLE_HISTS * 256; i += nthr) (&hist[0][0])[i] = 0;
      __syncthreads();
      const int b1 = pass ? s_sel[0] : 0;
      for (int i = tid; i < n_valid; i += nthr) {
        const uint32_t k = bf16_order_key(lr[i]);
        if (!k) continue;   // NaN
        if (pass == 0) atomicAdd(&myh[k >> 8], 1);
        else if ((int)(k >> 8) == b1) atomicAdd(&myh[k & 255u], 1);
      }
      __syncthreads();
      if (tid < 256) {
        int c = 0;
#pragma unroll
        for (int h = 0; h < SAMPLE_HISTS; ++h) c += hist[h][tid];
        hist[0][tid] = c;
      }
      __syncthreads();
      if (tid == 0) {
        int above = pass ? s_sel[1] : 0, b = 255;
        while (b > 0 && above + hist[0][b] < kk) { above += hist[0][b]; --b; }
        if (pass == 0) { s_sel[0] = b; s_sel[1] = above; }
        else { s_sel[2] = (s_sel[0] << 8) | b; s_sel[1] = above; s_sel[3] = 0; s_sel[4] = 0; }
      }
      __syncthreads();
    }
    const uint32_t thr = (uint32_t)s_sel[2];
    for (int i = tid; i < n_valid; i += nthr) {
      const bf16 v = lr[i];
      const uint32_t k = bf16_order_key(v);
      if (k && k >= thr) {
        const int slot = atomicAdd(&s_sel[3], 1);
        if (slot < SAMPLE_CAND) { cand_v[slot] = b2f(v); cand_i[slot] = i; }
      }
    }
    __syncthreads();
    if (s_sel[3] <= SAMPLE_CAND) { from_list = true; n_items = s_sel[3]; }   // else: massive ties at the threshold
  }

  if (big) {
    const uint32_t thr = (uint32_t)s_sel[2];
    const int above = s_sel[1];
    const int need = kk - above;          // ties at the threshold to take, lowest ids first
    const float inv_t = 1.0f / temp;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    if (from_list) {
      for (int t = tid; t < n_items; t += nthr) {
        const float v = cand_v[t];
        const int id = cand_i[t];
        bool in = bf16_order_key(f2b(v)) > thr;
        if (!in) {
          int rank = 0;
          for (int j = 0; j < n_items; ++j) rank += (cand_v[j] == v && cand_i[j] < id) ? 1 : 0;
          in = rank < need;
        }
        if (in) {
          const float sc = multinomial_score(v, inv_t, seed, stepc, (uint32_t)row, (uint32_t)id);
          if (sc > bv || (sc == bv && id < bi)) { bv = sc; bi = id; }
        }
      }
    } else {
      // more than SAMPLE_CAND logits share the threshold value: walk the row in index order, counting ties
      for (int base = 0; base < n_valid; base += nthr) {
        const int i = base + tid;
        const uint32_t k = i < n_valid ? bf16_order_key(lr[i]) : 0u;
        const bool tie = i < n_valid && k && k == thr;
        const unsigned bal = __ballot_sync(0xffffffffu, tie);
        const int wpre = __popc(bal & ((1u << (tid % 32)) - 1u));
        __syncthreads();
        if (tid % 32 == 0) s_idx[tid / 32] = __popc(bal);
        __syncthreads();
        int before = s_sel[4];
        for (int w = 0; w < tid / 32; ++w) before += s_idx[w];
        const bool in = i < n_valid && (k > thr || (tie && before + wpre < need));
        if (in) {
          const float sc = multinomial_score(b2f(lr[i]), inv_t, seed, stepc, (uint32_t)row, (uint32_t)i);
          if (sc > bv || (sc == bv && i < bi)) { bv = sc; bi = i; }
        }
        __syncthreads();
        if (tid == 0) { int t = 0; for (int w = 0; w < nthr / 32; ++w) t += s_idx[w]; s_sel[4] += t; }
        __syncthreads();
      }
    }
    block_argmax(bv, bi, s_val, s_idx);
    if (tid == 0) *token_out = bv > -INFINITY ? bi : 0;
    return;
  }

  float last_v = INFINITY;
  int last_i = -1;
  for (int r = 0; r < kk; ++r) {
    // largest (value, lowest index) strictly after (last_v, last_i) in the order (value desc, index asc)
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < n_items; i += nthr) {
      const float v = from_list ? cand_v[i] : b2f(lr[i]);
      const int id = from_list ? cand_i[i] : i;
      const bool after = v < last_v || (v == last_v && id > last_i);
      if (after && (v > bv || (v == bv && id < bi))) { bv = v; bi = id; }
    }
    block_argmax(bv, bi, s_val, s_idx);
    if (tid == 0) { top_v[r] = bv; top_i[r] = bi; }
    last_v = bv;
    last_i = bi;
  }
  if (tid == 0) {
    int pick = top_v[0] > -INFINITY ? top_i[0] : 0;   // no id above -inf (or none but NaN): id 0
    if (top_k > 0 && top_v[0] > -INFINITY) {
      float best = -INFINITY;
      for (int r = 0; r < kk && top_i[r] < n_valid; ++r) {   // (fewer than kk ids that are not NaN: the rest are empty)
        // a +inf logit weighs 1 (its difference to the top +inf would be NaN); then every other id weighs 0
        const float w = top_v[r] == INFINITY ? 1.f : expf((top_v[r] - top_v[0]) / temp);
        const uint32_t u = hash_u32(seed, stepc, (uint32_t)row, (uint32_t)r);
        const float uni = ((float)(u >> 8) + 0.5f) * (1.0f / 16777216.0f);  // (0,1)
        const float e = -logf(uni);                                        // Exp(1)
        const float score = w / e;
        if (score > best) { best = score; pick = top_i[r]; }
      }
    }
    *token_out = pick;
  }
}

// Per-row parameters (batches of utterances at different points of their generation): with step_rows set, row r draws
// its noise from (seed, step_rows[r], key_rows[r]) instead of (seed, *step_counter, r); with nvalid_rows set, its
// candidates are the ids < nvalid_rows[r * nv_stride] (top_k clamped to them as the host does for one n_valid).
// With topk_rows set (temp_rows and topp_rows with it), row r samples with top_k / temp / top_p from entry r * prm_stride
// of the three tables instead of the scalars; the host validates the tables, and the kernel clamps what would leave
// SAMPLE_CAND or the candidates (top_k), and reads temp <= 0 (or NaN) as argmax and a top_p that is not >= 0 as 0.
// Runtime branches around one call of the same sample_row body, so all forms draw identical tokens from identical inputs.
// Two 1 024-thread blocks per SM (32 registers, as before the nucleus mode; ptxas reports no spills).
__global__ void __launch_bounds__(1024, 2) sample_kernel(const bf16* __restrict__ logits, int V, int n_valid, int top_k, float temp, float top_p, uint32_t seed,
                              const long long* __restrict__ step_counter, long long* __restrict__ tokens, int tok_stride,
                              const int* __restrict__ nvalid_rows, int nv_stride, const long long* __restrict__ step_rows,
                              const uint32_t* __restrict__ key_rows, const int* __restrict__ topk_rows,
                              const float* __restrict__ temp_rows, const float* __restrict__ topp_rows, int prm_stride) {
  const int row = blockIdx.x;
  uint32_t stepc, key = (uint32_t)row;
  if (step_rows) {
    stepc = (uint32_t)step_rows[row];
    key = key_rows[row];
  } else {
    stepc = step_counter ? (uint32_t)(*step_counter) : 0u;
  }
  if (nvalid_rows) {
    n_valid = nvalid_rows[(long long)row * nv_stride];
    if (n_valid <= 0 || n_valid > V) n_valid = V;
    if (top_k > n_valid) top_k = n_valid;
  }
  if (topk_rows) {
    const long long o = (long long)row * prm_stride;
    top_k = topk_rows[o];
    temp = temp_rows[o];
    top_p = topp_rows[o];
    if (top_k > SAMPLE_CAND) top_k = SAMPLE_CAND;
    if (top_k > n_valid) top_k = n_valid;
    if (!(temp > 0.f)) { top_k = 0; temp = 1.f; }
    if (!(top_p >= 0.f)) top_p = 0.f;
  }
  sample_row(logits + (long long)row * V, n_valid, top_k, temp, top_p, seed, stepc, (int)key, tokens + (long long)row * tok_stride);
}

}  // namespace rstnet
using namespace rstnet;

extern "C" int rstnet_lm_embed_sum_bf16(const int64_t* seq, int32_t seq_stride, const void* wte, int64_t wte_rows,
                                        const void* const* tables_dev, int64_t table_rows, int32_t n_q, int32_t E, void* x,
                                        int32_t rows, rstnet_stream_t stream) {
  RSTNET_REQUIRE(seq && wte && tables_dev && x && rows > 0 && wte_rows > 0 && table_rows > 0, "lm_embed_sum: bad argument");
  embed_sum_kernel<<<dim3(rows), dim3(256), 0, (cudaStream_t)stream>>>((const long long*)seq, seq_stride, (const bf16*)wte,
             (const bf16* const*)tables_dev, n_q, E, (bf16*)x, (long long)wte_rows, (long long)table_rows);
  count_launch();
  return check_launch("lm_embed_sum");
}

extern "C" int rstnet_lm_embed_rows_bf16(const int64_t* ids, int32_t id_stride, const void* table, int64_t table_rows, int32_t D,
                                         void* out, int32_t rows, rstnet_stream_t stream) {
  RSTNET_REQUIRE(ids && table && out && rows > 0 && table_rows > 0, "lm_embed_rows: bad argument");
  embed_rows_kernel<<<dim3(rows), dim3(128), 0, (cudaStream_t)stream>>>((const long long*)ids, id_stride, (const bf16*)table, D,
             (bf16*)out, (long long)table_rows);
  count_launch();
  return check_launch("lm_embed_rows");
}

extern "C" int rstnet_lm_rms_norm_bf16(const void* x, const void* w, void* y, int32_t rows, int32_t dim, float eps, int32_t kyutai,
                                       rstnet_stream_t stream) {
  RSTNET_REQUIRE(x && w && y && rows > 0 && dim > 0, "lm_rms_norm: bad argument");
  rms_norm_kernel<<<dim3(rows), dim3(256), 0, (cudaStream_t)stream>>>((const bf16*)x, (const bf16*)w, (bf16*)y, dim, eps, kyutai);
  count_launch();
  return check_launch("lm_rms_norm");
}

// the page-table arguments of the paged entry points, checked before any launch
static int check_pages(const char* who, const int32_t* page_table, int32_t pages_stride, int32_t log2_page, int32_t cap) {
  RSTNET_REQUIRE(page_table, "%s: null page table", who);
  RSTNET_REQUIRE(log2_page >= RSTNET_KV_LOG2_PAGE_MIN && log2_page <= RSTNET_KV_LOG2_PAGE_MAX,
                 "%s: log2_page (%d) outside [%d, %d]", who, log2_page, RSTNET_KV_LOG2_PAGE_MIN, RSTNET_KV_LOG2_PAGE_MAX);
  RSTNET_REQUIRE(cap > 0 && pages_stride > 0 && ((long long)pages_stride << log2_page) >= cap,
                 "%s: pages_stride (%d) pages of %d positions do not cover the ring of %d", who, pages_stride, 1 << log2_page, cap);
  return 0;
}

static int rope_kv_append(const void* qkv, const void* cos_tab, const void* sin_tab, int64_t rope_rows, int32_t rope_n,
                          const int64_t* offset, int32_t offset_stride, const int32_t* row_stream, const int32_t* row_tl, void* q_out,
                          void* kv, int32_t rows, int32_t B, int32_t n_head, int32_t n_kv, int32_t hs, int32_t cap,
                          const int32_t* page_table, int32_t pages_stride, int32_t log2_page, rstnet_stream_t stream) {
  RSTNET_REQUIRE(qkv && cos_tab && sin_tab && offset && q_out && kv, "lm_rope_kv_append: null pointer");
  RSTNET_REQUIRE(!row_stream == !row_tl, "lm_rope_kv_append: row_stream and row_tl go together");
  RSTNET_REQUIRE(!row_stream || offset_stride, "lm_rope_kv_append: a row map needs per-stream offsets (offset_stride 1)");
  RSTNET_REQUIRE(rows > 0 && B > 0 && (row_stream || rows % B == 0),
                 "lm_rope_kv_append: rows (%d) must be a multiple of the stream count (%d) without a row map", rows, B);
  RSTNET_REQUIRE(n_kv > 0 && n_head % n_kv == 0, "lm_rope_kv_append: n_head (%d) must be a multiple of n_kv (%d)", n_head, n_kv);
  RSTNET_REQUIRE(rope_n >= 0 && rope_n <= hs && rope_n % 2 == 0 && rope_rows > 0, "lm_rope_kv_append: bad rope table (%d of %d dims)", rope_n, hs);
  rope_kv_append_bf16_kernel<<<dim3(rows * n_kv), dim3(64), 0, (cudaStream_t)stream>>>((const bf16*)qkv, (const bf16*)cos_tab,
             (const bf16*)sin_tab, (const long long*)offset, (bf16*)q_out, (bf16*)kv, offset_stride ? 1 : 0, B, n_kv, n_head / n_kv, hs,
             cap, rope_n, (long long)rope_rows, (const int*)row_stream, (const int*)row_tl, (const int*)page_table, pages_stride,
             log2_page);
  count_launch();
  return check_launch("lm_rope_kv_append");
}

extern "C" int rstnet_lm_rope_kv_append_bf16(const void* qkv, const void* cos_tab, const void* sin_tab, int64_t rope_rows,
                                             int32_t rope_n, const int64_t* offset, int32_t offset_stride, const int32_t* row_stream,
                                             const int32_t* row_tl, void* q_out, void* kv, int32_t rows, int32_t B, int32_t n_head,
                                             int32_t n_kv, int32_t hs, int32_t cap, rstnet_stream_t stream) {
  return rope_kv_append(qkv, cos_tab, sin_tab, rope_rows, rope_n, offset, offset_stride, row_stream, row_tl, q_out, kv, rows, B,
                        n_head, n_kv, hs, cap, nullptr, 0, 0, stream);
}

extern "C" int rstnet_lm_rope_kv_append_paged_bf16(const void* qkv, const void* cos_tab, const void* sin_tab, int64_t rope_rows,
                                                   int32_t rope_n, const int64_t* offset, int32_t offset_stride,
                                                   const int32_t* row_stream, const int32_t* row_tl, void* q_out, void* kv, int32_t rows,
                                                   int32_t B, int32_t n_head, int32_t n_kv, int32_t hs, int32_t cap,
                                                   const int32_t* page_table, int32_t pages_stride, int32_t log2_page,
                                                   rstnet_stream_t stream) {
  if (check_pages("lm_rope_kv_append_paged", page_table, pages_stride, log2_page, cap)) return 1;
  return rope_kv_append(qkv, cos_tab, sin_tab, rope_rows, rope_n, offset, offset_stride, row_stream, row_tl, q_out, kv, rows, B,
                        n_head, n_kv, hs, cap, page_table, pages_stride, log2_page, stream);
}

static int rope_pair_kv_append(const void* qkv, const int64_t* offset, int32_t offset_stride, void* q_out, void* kv, int32_t rows,
                               int32_t B, int32_t H, int32_t hd, int32_t cap, const float* freqs, const int32_t* page_table,
                               int32_t pages_stride, int32_t log2_page, const int32_t* row_stream, const int32_t* row_tl,
                               rstnet_stream_t stream) {
  RSTNET_REQUIRE(qkv && offset && q_out && kv && freqs, "lm_rope_pair_kv_append: null pointer");
  RSTNET_REQUIRE(rows > 0 && B > 0 && (row_stream || rows % B == 0) && H > 0 && hd > 0 && hd % 2 == 0 && cap > 0,
                 "lm_rope_pair_kv_append: bad shape");
  rope_pair_kv_append_bf16_kernel<<<dim3(rows * H), dim3(64), 0, (cudaStream_t)stream>>>((const bf16*)qkv,
             (const long long*)offset, offset_stride ? 1 : 0, (bf16*)q_out, (bf16*)kv, B, H, hd, cap, freqs, (const int*)page_table,
             pages_stride, log2_page, (const int*)row_stream, (const int*)row_tl);
  count_launch();
  return check_launch("lm_rope_pair_kv_append");
}

extern "C" int rstnet_lm_rope_pair_kv_append_bf16(const void* qkv, const int64_t* offset, int32_t offset_stride, void* q_out, void* kv,
                                                  int32_t rows, int32_t B, int32_t H, int32_t hd, int32_t cap, const float* freqs,
                                                  rstnet_stream_t stream) {
  return rope_pair_kv_append(qkv, offset, offset_stride, q_out, kv, rows, B, H, hd, cap, freqs, nullptr, 0, 0, nullptr, nullptr, stream);
}

extern "C" int rstnet_lm_rope_pair_kv_append_paged_bf16(const void* qkv, const int64_t* offset, int32_t offset_stride, void* q_out,
                                                        void* kv, int32_t rows, int32_t B, int32_t H, int32_t hd, int32_t cap,
                                                        const float* freqs, const int32_t* page_table, int32_t pages_stride,
                                                        int32_t log2_page, rstnet_stream_t stream) {
  if (check_pages("lm_rope_pair_kv_append_paged", page_table, pages_stride, log2_page, cap)) return 1;
  return rope_pair_kv_append(qkv, offset, offset_stride, q_out, kv, rows, B, H, hd, cap, freqs, page_table, pages_stride, log2_page,
                             nullptr, nullptr, stream);
}

extern "C" int rstnet_lm_rope_pair_kv_append_rows_bf16(const void* qkv, const int64_t* offset, const int32_t* row_stream,
                                                       const int32_t* row_tl, void* q_out, void* kv, int32_t rows, int32_t B, int32_t H,
                                                       int32_t hd, int32_t cap, const float* freqs, rstnet_stream_t stream) {
  RSTNET_REQUIRE(row_stream && row_tl, "lm_rope_pair_kv_append_rows: null row map");
  return rope_pair_kv_append(qkv, offset, 1, q_out, kv, rows, B, H, hd, cap, freqs, nullptr, 0, 0, row_stream, row_tl, stream);
}

extern "C" int rstnet_lm_rope_pair_kv_append_paged_rows_bf16(const void* qkv, const int64_t* offset, const int32_t* row_stream,
                                                             const int32_t* row_tl, void* q_out, void* kv, int32_t rows, int32_t B,
                                                             int32_t H, int32_t hd, int32_t cap, const float* freqs,
                                                             const int32_t* page_table, int32_t pages_stride, int32_t log2_page,
                                                             rstnet_stream_t stream) {
  RSTNET_REQUIRE(row_stream && row_tl, "lm_rope_pair_kv_append_paged_rows: null row map");
  if (check_pages("lm_rope_pair_kv_append_paged_rows", page_table, pages_stride, log2_page, cap)) return 1;
  return rope_pair_kv_append(qkv, offset, 1, q_out, kv, rows, B, H, hd, cap, freqs, page_table, pages_stride, log2_page, row_stream,
                             row_tl, stream);
}

static int ring_decode_attention(const void* q, const void* kv, const int64_t* offset, int32_t offset_stride,
                                 const int32_t* row_stream, const int32_t* row_tl, void* out, int32_t rows, int32_t B, int32_t n_head,
                                 int32_t n_kv, int32_t hs, int32_t cap, int32_t context, const int32_t* page_table,
                                 int32_t pages_stride, int32_t log2_page, rstnet_stream_t stream) {
  RSTNET_REQUIRE(q && kv && offset && out, "lm_ring_decode_attention: null pointer");
  RSTNET_REQUIRE(!row_stream == !row_tl, "lm_ring_decode_attention: row_stream and row_tl go together");
  RSTNET_REQUIRE(!row_stream || offset_stride, "lm_ring_decode_attention: a row map needs per-stream offsets (offset_stride 1)");
  RSTNET_REQUIRE(hs == 128 || hs == 64, "lm_ring_decode_attention: head_size must be 64 or 128 (got %d)", hs);
  RSTNET_REQUIRE(rows > 0 && B > 0 && (row_stream || rows % B == 0),
                 "lm_ring_decode_attention: rows (%d) must be a multiple of the stream count (%d) without a row map", rows, B);
  RSTNET_REQUIRE(n_kv > 0 && n_head % n_kv == 0, "lm_ring_decode_attention: n_head (%d) must be a multiple of n_kv (%d)", n_head, n_kv);
  // the window of a query is max(0, pos - context + 1, pos + 2 - cap) .. pos: with cap < 2 or context < 1 it is empty and
  // every output would be 0 / 0
  RSTNET_REQUIRE(cap >= 2 && context >= 1, "lm_ring_decode_attention: cap (%d) must be >= 2 and context (%d) >= 1", cap, context);
  const float scale = 1.0f / sqrtf((float)hs);
  const int q_per_kv = n_head / n_kv;
  const int G = q_per_kv % 2 == 0 ? 2 : 1;   // query heads per CTA sharing the K/V rows (the rest of a group hits L2)
  const auto launch = hs == 128 ? (G == 2 ? launch_ring_decode_attention<128, 2> : launch_ring_decode_attention<128, 1>)
                                : (G == 2 ? launch_ring_decode_attention<64, 2> : launch_ring_decode_attention<64, 1>);
  launch((cudaStream_t)stream, (const bf16*)q, (const bf16*)kv, (const long long*)offset, (bf16*)out, offset_stride ? 1 : 0, rows, B,
         n_head, n_kv, cap, context, scale, (const int*)row_stream, (const int*)row_tl, (const int*)page_table, pages_stride, log2_page);
  count_launch();
  return check_launch("lm_ring_decode_attention");
}

extern "C" int rstnet_lm_ring_decode_attention_bf16(const void* q, const void* kv, const int64_t* offset, int32_t offset_stride,
                                                    const int32_t* row_stream, const int32_t* row_tl, void* out, int32_t rows,
                                                    int32_t B, int32_t n_head, int32_t n_kv, int32_t hs, int32_t cap, int32_t context,
                                                    rstnet_stream_t stream) {
  return ring_decode_attention(q, kv, offset, offset_stride, row_stream, row_tl, out, rows, B, n_head, n_kv, hs, cap, context, nullptr,
                               0, 0, stream);
}

extern "C" int rstnet_lm_paged_decode_attention_bf16(const void* q, const void* kv, const int64_t* offset, int32_t offset_stride,
                                                     const int32_t* row_stream, const int32_t* row_tl, void* out, int32_t rows,
                                                     int32_t B, int32_t n_head, int32_t n_kv, int32_t hs, int32_t cap, int32_t context,
                                                     const int32_t* page_table, int32_t pages_stride, int32_t log2_page,
                                                     rstnet_stream_t stream) {
  if (check_pages("lm_paged_decode_attention", page_table, pages_stride, log2_page, cap)) return 1;
  return ring_decode_attention(q, kv, offset, offset_stride, row_stream, row_tl, out, rows, B, n_head, n_kv, hs, cap, context,
                               page_table, pages_stride, log2_page, stream);
}

extern "C" int rstnet_lm_silu_mul_bf16(const void* ab, void* out, int32_t M, int32_t I, rstnet_stream_t stream) {
  RSTNET_REQUIRE(ab && out && M > 0 && I > 0, "lm_silu_mul: bad argument");
  const long long total = (long long)M * I;
  int g = ceil_div(total, 256);
  if (g > sm_count() * 8) g = sm_count() * 8;
  silu_mul_kernel<<<dim3(g), dim3(256), 0, (cudaStream_t)stream>>>((const bf16*)ab, (bf16*)out, M, I);
  count_launch();
  return check_launch("lm_silu_mul");
}

extern "C" int rstnet_lm_depth_attention_bf16(const void* qkv, void* kvd, void* out, int32_t B, int32_t H, int32_t hd, int32_t cap,
                                              int32_t step, int32_t ring_quirk, rstnet_stream_t stream) {
  RSTNET_REQUIRE(qkv && kvd && out, "lm_depth_attention: null pointer");
  RSTNET_REQUIRE(step >= 0 && step < cap && cap <= 8, "lm_depth_attention: step %d / capacity %d (<= 8) out of range", step, cap);
  depth_attention_kernel<<<dim3(B * H), dim3(32), 0, (cudaStream_t)stream>>>((const bf16*)qkv, (bf16*)kvd, (bf16*)out, B, H, hd, cap,
             step, ring_quirk);
  count_launch();
  return check_launch("lm_depth_attention");
}

// ---------------------------------------------------------------- forced tokens (generation with given ids)
// tokens[r, col] = force[r, col] where that id is >= 0; a negative id keeps the sample.  An id >= V is not written: it
// sets error bit 0 (1), as an out-of-range embedding id does.  One thread per row.
__global__ void force_tokens_kernel(long long* __restrict__ tokens, int tok_stride, int col, const int* __restrict__ force,
                                    int force_stride, int rows, int V) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int id = force[(long long)r * force_stride + col];
  if (id < 0) return;
  if (id >= V) {
    atomicOr(&g_lm_dev_err, 1u);
    return;
  }
  tokens[(long long)r * tok_stride + col] = id;
}

extern "C" int rstnet_lm_force_tokens(int64_t* tokens, int32_t tok_stride, int32_t col, const int32_t* force, int32_t force_stride,
                                      int32_t rows, int32_t V, rstnet_stream_t stream) {
  RSTNET_REQUIRE(tokens && force, "lm_force_tokens: null pointer");
  RSTNET_REQUIRE(rows > 0 && V > 0 && col >= 0 && col < tok_stride && col < force_stride,
                 "lm_force_tokens: bad shape (rows=%d, V=%d, col=%d, tok_stride=%d, force_stride=%d)", rows, V, col, tok_stride,
                 force_stride);
  force_tokens_kernel<<<dim3(ceil_div(rows, 256)), dim3(256), 0, (cudaStream_t)stream>>>((long long*)tokens, tok_stride, col, force,
                                                                                          force_stride, rows, V);
  count_launch();
  return check_launch("lm_force_tokens");
}

extern "C" int rstnet_lm_sample_params_bf16(const void* logits, int32_t rows, int32_t V, int32_t n_valid, const int32_t* n_valid_rows,
                                            int32_t n_valid_stride, int32_t top_k, float temp, float top_p, const int32_t* top_k_rows,
                                            const float* temp_rows, const float* top_p_rows, int32_t param_stride, uint32_t seed,
                                            const int64_t* step_counter, const int64_t* step_rows, const uint32_t* key_rows,
                                            int64_t* tokens, int32_t tok_stride, rstnet_stream_t stream) {
  RSTNET_REQUIRE(logits && tokens && rows > 0 && V > 0, "lm_sample_params: bad argument");
  const bool tables = top_k_rows || temp_rows || top_p_rows;
  RSTNET_REQUIRE(!tables || (top_k_rows && temp_rows && top_p_rows && param_stride > 0),
                 "lm_sample_params: the top_k / temp / top_p tables go together, with a stride > 0");
  RSTNET_REQUIRE(!step_rows == !key_rows, "lm_sample_params: step_rows and key_rows go together");
  RSTNET_REQUIRE(!n_valid_rows || n_valid_stride > 0, "lm_sample_params: n_valid_rows needs a stride > 0");
  if (!tables) {
    RSTNET_REQUIRE(top_k <= SAMPLE_CAND && (top_k == 0 || temp > 0.f), "lm_sample_params: top_k <= %d and temp > 0 required (top_k=%d)",
                   SAMPLE_CAND, top_k);
    RSTNET_REQUIRE(isfinite(top_p) && top_p >= 0.f, "lm_sample_params: top_p must be finite and >= 0 (got %g)", (double)top_p);
  }
  if (n_valid <= 0 || n_valid > V) n_valid = V;
  if (!n_valid_rows && top_k > n_valid) top_k = n_valid;   // with per-row candidate counts the kernel clamps per row
  sample_kernel<<<dim3(rows), dim3(1024), 0, (cudaStream_t)stream>>>((const bf16*)logits, V, n_valid, top_k, temp, top_p, (uint32_t)seed,
             (const long long*)step_counter, (long long*)tokens, tok_stride, (const int*)n_valid_rows, n_valid_stride,
             (const long long*)step_rows, key_rows, (const int*)top_k_rows, temp_rows, top_p_rows, param_stride);
  count_launch();
  return check_launch("lm_sample_params");
}
