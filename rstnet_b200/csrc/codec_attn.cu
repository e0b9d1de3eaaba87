// Codec transformer attention: pair-RoPE + ring-KV append, then masked ring attention.
// Follows StreamingMultiheadAttention.forward (modules/transformer.py:375-419), apply_rope
// (modules/rope.py:11-68) and RingKVCache.complete (transformer.py:211-278) of the reference.
// HBM/L2-bound gather work (0.05 GMAC per stream-second): CUDA cores, one warp per query.
#include <cstdint>

#include "common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {
extern void count_launch();

// cos / sin of a RoPE angle, out of line: the separate append kernel and the fused attention kernel must rotate bit for
// bit alike, and inlined copies of cosf / sinf may be contracted or share their range reduction differently per call site
__device__ __noinline__ float2 rope_cos_sin(float ang) { return make_float2(cosf(ang), sinf(ang)); }

// one warp per (b, t, h); lanes stride over the D/2 rotation pairs
__global__ void rope_kv_append_kernel(float* __restrict__ qkv, long long qbs, long long qts, float* __restrict__ kv,
                                      const long long* __restrict__ offset, int ostride, const float* __restrict__ freqs,
                                      int B, int T, int H, int D, int cap) {
  const long long wid = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  const long long total = (long long)B * T * H;
  if (wid >= total) return;
  const int h = (int)(wid % H);
  const int t = (int)((wid / H) % T);
  const int b = (int)(wid / ((long long)H * T));
  const long long off = offset[(long long)b * ostride];   // per-stream position counters (ostride 1) or one shared (0)
  const long long pos = off + t;
  const int slot = (int)(pos % cap);
  const int HD = H * D;
  float* q = qkv + b * qbs + t * qts + h * D;
  float* k = q + HD;
  const float* v = q + 2 * HD;
  float* kdst = kv + (((long long)b * H + h) * cap + slot) * D;
  float* vdst = kv + (long long)B * H * cap * D + (((long long)b * H + h) * cap + slot) * D;
  // ts = offset.float() + arange(T) in fp32 (rope.py:39)
  const float ts = __fadd_rn((float)off, (float)t);
  for (int pr = lane; pr < D / 2; pr += 32) {
    const float2 cs = rope_cos_sin(__fmul_rn(freqs[pr], ts));
    const float c = cs.x, s = cs.y;
    const float qr = q[2 * pr], qi = q[2 * pr + 1];
    const float kr = k[2 * pr], ki = k[2 * pr + 1];
    // separate mul / sub / add (no FMA contraction) as the eager reference evaluates them
    q[2 * pr] = __fsub_rn(__fmul_rn(qr, c), __fmul_rn(qi, s));
    q[2 * pr + 1] = __fadd_rn(__fmul_rn(qr, s), __fmul_rn(qi, c));
    kdst[2 * pr] = __fsub_rn(__fmul_rn(kr, c), __fmul_rn(ki, s));
    kdst[2 * pr + 1] = __fadd_rn(__fmul_rn(kr, s), __fmul_rn(ki, c));
    vdst[2 * pr] = v[2 * pr];
    vdst[2 * pr + 1] = v[2 * pr + 1];
  }
}

// one warp per (b, h, tq): lane j scores key j of each 32-key block, online softmax, then the
// lanes own output dims (lane, lane+32, ...) for the P.V accumulation (coalesced V reads).
__global__ void ring_attention_kernel(const float* __restrict__ qkv, long long qbs, long long qts,
                                      const float* __restrict__ kv, const long long* __restrict__ offset, int ostride,
                                      float* __restrict__ out, long long obs, long long ots, int B, int T, int H, int D, int cap,
                                      int context, int linear) {
  extern __shared__ __align__(16) float qs_all[];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const long long wid = (long long)blockIdx.x * (blockDim.x / 32) + warp;
  const long long total = (long long)B * T * H;
  float* qs = qs_all + warp * D;
  const bool active = wid < total;
  int h = 0, t = 0, b = 0;
  if (active) {
    h = (int)(wid % H);
    t = (int)((wid / H) % T);
    b = (int)(wid / ((long long)H * T));
    const float* q = qkv + b * qbs + t * qts + h * D;
    for (int d = lane; d < D; d += 32) qs[d] = q[d];
  }
  __syncwarp();
  if (!active) return;
  const long long off = offset[(long long)b * ostride];
  const long long end = off + T;
  const long long pos_q = off + t;
  long long lo = pos_q - context + 1;
  if (lo < 0) lo = 0;
  // RingKVCache.complete (transformer.py:258-263) labels the slot at end_offset % capacity with
  // position `end_offset` (its `delta <= 0` branch), so once the ring has wrapped the oldest entry
  // (position end - cap) is masked out by `delta >= 0`: only cap - 1 keys are attendable.
  // A linear (non-streaming, KVCacheResult.from_kv) buffer keeps every position.
  if (!linear && lo < end - cap + 1) lo = end - cap + 1;
  const float* Kb = kv + ((long long)b * H + h) * cap * D;
  const float* Vb = Kb + (long long)B * H * cap * D;
  const float scale = 1.0f / sqrtf((float)D);
  float m = -INFINITY, l = 0.f;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long p0 = lo; p0 <= pos_q; p0 += 32) {
    const long long p = p0 + lane;
    const bool valid = p <= pos_q;
    const int slot = (int)((valid ? p : pos_q) % cap);
    float s = -INFINITY;
    if (valid) {
      const float4* kp = reinterpret_cast<const float4*>(Kb + (long long)slot * D);
      const float4* qp = reinterpret_cast<const float4*>(qs);
      float dot = 0.f;
      for (int d4 = 0; d4 < D / 4; ++d4) {
        const float4 kk = kp[d4], qq = qp[d4];
        dot = fmaf(qq.x, kk.x, dot); dot = fmaf(qq.y, kk.y, dot);
        dot = fmaf(qq.z, kk.z, dot); dot = fmaf(qq.w, kk.w, dot);
      }
      s = dot * scale;
    }
    const float m_new = fmaxf(m, warp_max(s));
    const float corr = expf(m - m_new);  // exp(-inf) = 0 on the first block
    const float pj = valid ? expf(s - m_new) : 0.f;
    l = l * corr + warp_sum(pj);
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i] *= corr;
    const int nk = (int)min(32LL, pos_q - p0 + 1);
    for (int j = 0; j < nk; ++j) {
      const float pw = __shfl_sync(0xffffffffu, pj, j);
      const int sj = __shfl_sync(0xffffffffu, slot, j);
      const float* vp = Vb + (long long)sj * D;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int d = lane + 32 * i;
        if (d < D) acc[i] = fmaf(pw, vp[d], acc[i]);
      }
    }
    m = m_new;
  }
  float* o = out + b * obs + t * ots + h * D;
  const float inv = 1.0f / l;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int d = lane + 32 * i;
    if (d < D) o[d] = acc[i] * inv;
  }
}


// Two consecutive queries (2k, 2k+1) of one (b, h) per warp: a streaming step carries exactly one such pair per
// stream (two 25 Hz tokens per 80 ms frame), and the pair shares every K / V row it reads -- at a full 250-token
// context the fp32 ring (64 KB of K + 64 KB of V per (b, h)) is the HBM traffic of this kernel, so reading it once
// instead of twice halves it.  Per query the arithmetic is the single-query kernel's (same block walk from the
// pair's first key, same FMA order); a query that ends before the block gets zero weights there.
__global__ void ring_attention_pair_kernel(const float* __restrict__ qkv, long long qbs, long long qts,
                                           const float* __restrict__ kv, const long long* __restrict__ offset, int ostride,
                                           float* __restrict__ out, long long obs, long long ots, int B, int T, int H, int D,
                                           int cap, int context, int linear) {
  extern __shared__ __align__(16) float qs_all[];
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int P = (T + 1) / 2;
  const long long wid = (long long)blockIdx.x * (blockDim.x / 32) + warp;
  const long long total = (long long)B * P * H;
  float* qs0 = qs_all + warp * 2 * D;
  float* qs1 = qs0 + D;
  if (wid >= total) return;
  const int h = (int)(wid % H);
  const int t0 = 2 * (int)((wid / H) % P);
  const int b = (int)(wid / ((long long)H * P));
  const bool has1 = t0 + 1 < T;
  {
    const float* q0 = qkv + b * qbs + t0 * qts + h * D;
    const float* q1 = has1 ? q0 + qts : q0;
    for (int d = lane; d < D; d += 32) { qs0[d] = q0[d]; qs1[d] = q1[d]; }
  }
  __syncwarp();
  const long long off = offset[(long long)b * ostride];
  const long long end = off + T;
  const long long pos0 = off + t0, pos1 = has1 ? pos0 + 1 : pos0;
  long long lo0 = pos0 - context + 1, lo1 = pos1 - context + 1;
  if (lo0 < 0) lo0 = 0;
  if (lo1 < 0) lo1 = 0;
  if (!linear) {   // ring quirk, see ring_attention_kernel
    if (lo0 < end - cap + 1) lo0 = end - cap + 1;
    if (lo1 < end - cap + 1) lo1 = end - cap + 1;
  }
  const float* Kb = kv + ((long long)b * H + h) * cap * D;
  const float* Vb = Kb + (long long)B * H * cap * D;
  const float scale = 1.0f / sqrtf((float)D);
  float m0 = -INFINITY, l0 = 0.f, m1 = -INFINITY, l1 = 0.f;
  float acc0[4] = {0.f, 0.f, 0.f, 0.f}, acc1[4] = {0.f, 0.f, 0.f, 0.f};
  for (long long p0 = lo0; p0 <= pos1; p0 += 32) {
    const long long p = p0 + lane;
    const bool in = p <= pos1;
    const bool v0 = p <= pos0, v1 = in && p >= lo1;
    const int slot = (int)((in ? p : pos1) % cap);
    float s0 = -INFINITY, s1 = -INFINITY;
    if (in) {
      const float4* kp = reinterpret_cast<const float4*>(Kb + (long long)slot * D);
      const float4* qa = reinterpret_cast<const float4*>(qs0);
      const float4* qb = reinterpret_cast<const float4*>(qs1);
      float d0 = 0.f, d1 = 0.f;
      for (int d4 = 0; d4 < D / 4; ++d4) {
        const float4 kk = kp[d4], a = qa[d4], c = qb[d4];
        d0 = fmaf(a.x, kk.x, d0); d0 = fmaf(a.y, kk.y, d0); d0 = fmaf(a.z, kk.z, d0); d0 = fmaf(a.w, kk.w, d0);
        d1 = fmaf(c.x, kk.x, d1); d1 = fmaf(c.y, kk.y, d1); d1 = fmaf(c.z, kk.z, d1); d1 = fmaf(c.w, kk.w, d1);
      }
      if (v0) s0 = d0 * scale;
      if (v1) s1 = d1 * scale;
    }
    const float m0n = fmaxf(m0, warp_max(s0)), m1n = fmaxf(m1, warp_max(s1));
    const float c0 = expf(m0 - m0n), c1 = expf(m1 - m1n);   // exp(-inf) = 0 on a query's first block
    const float pj0 = v0 ? expf(s0 - m0n) : 0.f, pj1 = v1 ? expf(s1 - m1n) : 0.f;
    l0 = l0 * c0 + warp_sum(pj0);
    l1 = l1 * c1 + warp_sum(pj1);
#pragma unroll
    for (int i = 0; i < 4; ++i) { acc0[i] *= c0; acc1[i] *= c1; }
    const int nk = (int)min(32LL, pos1 - p0 + 1);
    for (int j = 0; j < nk; ++j) {
      const float w0 = __shfl_sync(0xffffffffu, pj0, j), w1 = __shfl_sync(0xffffffffu, pj1, j);
      const int sj = __shfl_sync(0xffffffffu, slot, j);
      const float* vp = Vb + (long long)sj * D;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int d = lane + 32 * i;
        if (d < D) { const float vv = vp[d]; acc0[i] = fmaf(w0, vv, acc0[i]); acc1[i] = fmaf(w1, vv, acc1[i]); }
      }
    }
    m0 = m0n; m1 = m1n;
  }
  float* o0 = out + b * obs + t0 * ots + h * D;
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int d = lane + 32 * i;
    if (d < D) { o0[d] = acc0[i] * i0; if (has1) o0[ots + d] = acc1[i] * i1; }
  }
}


// head_dim 64 version of the pair kernel with coalesced traffic.  K: eight lanes share one key row (each lane owns eight
// of the 64 dims, its two query slices live in registers), so a 128-bit load instruction covers four whole rows
// instead of 32 different lines; the partial dots are reduced with three shuffles.  V: sixteen lanes cover one row with
// 128-bit loads (two rows per instruction), the two half-warps accumulate alternate keys and are added at the end.
// Ring slots advance incrementally (no per-key modulo).  The one-row-per-lane form read 32 different lines per load
// instruction and was the slowest launch of a late streaming frame.
// ROPE: the streaming step (T == 2: one warp owns both new tokens of its (stream, head)) rotates q in registers, rotates and
// appends k, copies v into the ring itself -- arithmetic of rope_kv_append_kernel above -- and then attends; the separate
// RoPE / append launch (16 per frame) disappears.  The ring is read with plain loads (the warp may read rows it wrote).
// The fused form (freqs != nullptr) is a runtime branch of ONE compiled kernel, not a second instantiation: both forms then
// run the same attention instructions, so they agree bit for bit whatever FMA contraction the compiler chooses.
__global__ void __launch_bounds__(128, 4) ring_attention_pair64_kernel(const float* __restrict__ qkv, long long qbs, long long qts,
                                             float* kv, const long long* __restrict__ offset, int ostride,
                                             float* __restrict__ out, long long obs, long long ots, int B, int T, int H,
                                             int cap, int context, int linear, const float* __restrict__ freqs) {
  constexpr int D = 64;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int P = (T + 1) / 2;
  const long long wid = (long long)blockIdx.x * (blockDim.x / 32) + warp;
  if (wid >= (long long)B * P * H) return;
  const int h = (int)(wid % H);
  const int t0 = 2 * (int)((wid / H) % P);
  const int b = (int)(wid / ((long long)H * P));
  const bool has1 = t0 + 1 < T;
  const int grp = lane >> 3, sub = lane & 7;       // K phase: key = 4 * it + grp, dims [8 sub, 8 sub + 8)
  const int half = lane >> 4, vl = lane & 15;       // V phase: key = 2 * i + half, dims [4 vl, 4 vl + 4)
  float qa[8], qb[8];
  {
    const float* q0 = qkv + b * qbs + t0 * qts + h * D + 8 * sub;
    const float* q1 = has1 ? q0 + qts : q0;
    const float4 a0 = *reinterpret_cast<const float4*>(q0), a1 = *reinterpret_cast<const float4*>(q0 + 4);
    const float4 b0 = *reinterpret_cast<const float4*>(q1), b1 = *reinterpret_cast<const float4*>(q1 + 4);
    qa[0] = a0.x; qa[1] = a0.y; qa[2] = a0.z; qa[3] = a0.w; qa[4] = a1.x; qa[5] = a1.y; qa[6] = a1.z; qa[7] = a1.w;
    qb[0] = b0.x; qb[1] = b0.y; qb[2] = b0.z; qb[3] = b0.w; qb[4] = b1.x; qb[5] = b1.y; qb[6] = b1.z; qb[7] = b1.w;
  }
  const long long off = offset[(long long)b * ostride];
  const long long end = off + T;
  const long long pos0 = off + t0, pos1 = has1 ? pos0 + 1 : pos0;
  if (freqs) {
    // ts = offset.float() + arange(T) in fp32 (rope.py:39); separate mul / sub / add as the eager reference evaluates them
    auto rotate8 = [&](float* x, float ts) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 cs = rope_cos_sin(__fmul_rn(freqs[4 * sub + i], ts));
        const float c = cs.x, s = cs.y;
        const float xr = x[2 * i], xi = x[2 * i + 1];
        x[2 * i] = __fsub_rn(__fmul_rn(xr, c), __fmul_rn(xi, s));
        x[2 * i + 1] = __fadd_rn(__fmul_rn(xr, s), __fmul_rn(xi, c));
      }
    };
    rotate8(qa, __fadd_rn((float)off, (float)t0));
    if (has1) rotate8(qb, __fadd_rn((float)off, (float)(t0 + 1)));
    else {
#pragma unroll
      for (int i = 0; i < 8; ++i) qb[i] = qa[i];
    }
    // lanes 0-7 / 8-15: k of token t0 / t0+1 (rotated), lanes 16-23 / 24-31: v of token t0 / t0+1
    const int tok = grp & 1, is_v = grp >> 1;
    if (tok == 0 || has1) {
      const int HD = H * D;
      const float* src = qkv + b * qbs + (long long)(t0 + tok) * qts + h * D + (is_v ? 2 * HD : HD) + 8 * sub;
      const float4 s0 = *reinterpret_cast<const float4*>(src), s1 = *reinterpret_cast<const float4*>(src + 4);
      float x[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
      if (!is_v) rotate8(x, __fadd_rn((float)off, (float)(t0 + tok)));
      const int slot = (int)((pos0 + tok) % cap);
      float* dst = kv + (is_v ? (long long)B * H * cap * D : 0) + (((long long)b * H + h) * cap + slot) * D + 8 * sub;
      *reinterpret_cast<float4*>(dst) = make_float4(x[0], x[1], x[2], x[3]);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(x[4], x[5], x[6], x[7]);
    }
    __syncwarp();
  }
  long long lo0 = pos0 - context + 1, lo1 = pos1 - context + 1;
  if (lo0 < 0) lo0 = 0;
  if (lo1 < 0) lo1 = 0;
  if (!linear) {   // ring quirk, see ring_attention_kernel
    if (lo0 < end - cap + 1) lo0 = end - cap + 1;
    if (lo1 < end - cap + 1) lo1 = end - cap + 1;
  }
  const float* Kb = kv + ((long long)b * H + h) * cap * D;
  const float* Vb = Kb + (long long)B * H * cap * D;
  const float scale = 0.125f;   // 1 / sqrt(64)
  float m0 = -INFINITY, l0 = 0.f, m1 = -INFINITY, l1 = 0.f;
  float4 acc0 = make_float4(0.f, 0.f, 0.f, 0.f), acc1 = acc0;
  const int slot_last = (int)(pos1 % cap);
  const bool small_ring = cap < 32;        // uniform: short non-streaming clips (cap == T) and test rings
  for (long long p0 = lo0; p0 <= pos1; p0 += 32) {
    const int base = (int)(p0 % cap);
    // ---- scores of the 32 keys of the block: lane holds keys 4 it + grp, it = 0..7
    // All 16 K loads of the block are issued before the first use (branch-free slot arithmetic keeps the unrolled loop
    // one basic block): with a `while (slot >= cap)` wrap per key the compiler could keep only two loads in flight per
    // warp and the kernel ran at memory LATENCY, not bandwidth.
    float s0[8], s1[8];
    {
      float4 kq[8][2];
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        int slot = base + 4 * it + grp;               // base < cap and 4 it + grp < 32: one wrap unless the ring is tiny
        slot = small_ring ? slot % cap : (slot >= cap ? slot - cap : slot);
        const bool in = p0 + 4 * it + grp <= pos1;
        const float* kr = Kb + (long long)(in ? slot : slot_last) * D + 8 * sub;
        kq[it][0] = *reinterpret_cast<const float4*>(kr);
        kq[it][1] = *reinterpret_cast<const float4*>(kr + 4);
      }
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const long long p = p0 + 4 * it + grp;
        const bool in = p <= pos1;
        const float4 k0 = kq[it][0], k1 = kq[it][1];
        float d0 = qa[0] * k0.x, d1 = qb[0] * k0.x;
        d0 = fmaf(qa[1], k0.y, d0); d0 = fmaf(qa[2], k0.z, d0); d0 = fmaf(qa[3], k0.w, d0);
        d0 = fmaf(qa[4], k1.x, d0); d0 = fmaf(qa[5], k1.y, d0); d0 = fmaf(qa[6], k1.z, d0); d0 = fmaf(qa[7], k1.w, d0);
        d1 = fmaf(qb[1], k0.y, d1); d1 = fmaf(qb[2], k0.z, d1); d1 = fmaf(qb[3], k0.w, d1);
        d1 = fmaf(qb[4], k1.x, d1); d1 = fmaf(qb[5], k1.y, d1); d1 = fmaf(qb[6], k1.z, d1); d1 = fmaf(qb[7], k1.w, d1);
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) { d0 += __shfl_xor_sync(0xffffffffu, d0, o); d1 += __shfl_xor_sync(0xffffffffu, d1, o); }
        s0[it] = (p <= pos0) ? d0 * scale : -INFINITY;                 // p >= lo0 by construction
        s1[it] = (in && p >= lo1) ? d1 * scale : -INFINITY;
      }
    }
    float bm0 = s0[0], bm1 = s1[0];
#pragma unroll
    for (int it = 1; it < 8; ++it) { bm0 = fmaxf(bm0, s0[it]); bm1 = fmaxf(bm1, s1[it]); }
    const float m0n = fmaxf(m0, warp_max(bm0)), m1n = fmaxf(m1, warp_max(bm1));
    const float c0 = expf(m0 - m0n), c1 = expf(m1 - m1n);   // exp(-inf) = 0 on a query's first block
    float ps0 = 0.f, ps1 = 0.f;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      s0[it] = s0[it] == -INFINITY ? 0.f : expf(s0[it] - m0n);
      s1[it] = s1[it] == -INFINITY ? 0.f : expf(s1[it] - m1n);
      ps0 += s0[it]; ps1 += s1[it];
    }
    if (sub != 0) { ps0 = 0.f; ps1 = 0.f; }   // the eight lanes of a group hold the same weights: count them once
    l0 = l0 * c0 + warp_sum(ps0);
    l1 = l1 * c1 + warp_sum(ps1);
    acc0.x *= c0; acc0.y *= c0; acc0.z *= c0; acc0.w *= c0;
    acc1.x *= c1; acc1.y *= c1; acc1.z *= c1; acc1.w *= c1;
    // ---- P.V: half-warp `half` takes keys 2 i + half
    // keys past the pair's last position carry zero weights, so their V loads are redirected to the last valid row
    // (finite values) instead of being skipped: all 16 loads go out together, no per-key branch
    const int nk = (int)min(32LL, pos1 - p0 + 1);
    float4 vq[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int j = 2 * i + half;
      int slot = base + j;
      slot = small_ring ? slot % cap : (slot >= cap ? slot - cap : slot);
      vq[i] = *reinterpret_cast<const float4*>(Vb + (long long)(j < nk ? slot : slot_last) * D + 4 * vl);
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      // key j = 2 i + half lives at register index j / 4 of the lanes of group j % 4
      const int src = (((2 * i) & 3) + half) << 3;
      const float w0 = __shfl_sync(0xffffffffu, s0[i >> 1], src), w1 = __shfl_sync(0xffffffffu, s1[i >> 1], src);
      const float4 vv = vq[i];
      acc0.x = fmaf(w0, vv.x, acc0.x); acc0.y = fmaf(w0, vv.y, acc0.y); acc0.z = fmaf(w0, vv.z, acc0.z); acc0.w = fmaf(w0, vv.w, acc0.w);
      acc1.x = fmaf(w1, vv.x, acc1.x); acc1.y = fmaf(w1, vv.y, acc1.y); acc1.z = fmaf(w1, vv.z, acc1.z); acc1.w = fmaf(w1, vv.w, acc1.w);
    }
    m0 = m0n; m1 = m1n;
  }
  // even keys + odd keys
  acc0.x += __shfl_xor_sync(0xffffffffu, acc0.x, 16); acc0.y += __shfl_xor_sync(0xffffffffu, acc0.y, 16);
  acc0.z += __shfl_xor_sync(0xffffffffu, acc0.z, 16); acc0.w += __shfl_xor_sync(0xffffffffu, acc0.w, 16);
  acc1.x += __shfl_xor_sync(0xffffffffu, acc1.x, 16); acc1.y += __shfl_xor_sync(0xffffffffu, acc1.y, 16);
  acc1.z += __shfl_xor_sync(0xffffffffu, acc1.z, 16); acc1.w += __shfl_xor_sync(0xffffffffu, acc1.w, 16);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
  float* o0 = out + b * obs + t0 * ots + h * D + 4 * vl;
  if (half == 0) *reinterpret_cast<float4*>(o0) = make_float4(acc0.x * i0, acc0.y * i0, acc0.z * i0, acc0.w * i0);
  else if (has1) *reinterpret_cast<float4*>(o0 + ots) = make_float4(acc1.x * i1, acc1.y * i1, acc1.z * i1, acc1.w * i1);
}

}  // namespace rstnet
using namespace rstnet;

extern "C" int rstnet_rope_kv_append_f32(float* qkv, int64_t q_batch_stride, int64_t q_time_stride, float* kv,
                                         const int64_t* offset, int32_t offset_stride, const float* freqs, int32_t batch,
                                         int32_t T, int32_t H, int32_t D, int32_t cap, rstnet_stream_t stream) {
  RSTNET_REQUIRE(qkv && kv && offset && freqs, "rope_kv_append: null pointer");
  RSTNET_REQUIRE(batch > 0 && T > 0 && H > 0 && D > 0 && D % 2 == 0 && cap > 0, "rope_kv_append: bad shape");
  RSTNET_REQUIRE(T <= cap, "rope_kv_append: T (%d) exceeds ring capacity (%d)", T, cap);
  const long long total = (long long)batch * T * H;
  const int warps = 8;
  rope_kv_append_kernel<<<ceil_div(total, warps), warps * 32, 0, (cudaStream_t)stream>>>(
      qkv, q_batch_stride, q_time_stride, kv, (const long long*)offset, offset_stride ? 1 : 0, freqs, batch, T, H, D, cap);
  count_launch();
  return check_launch("rope_kv_append");
}

extern "C" int rstnet_rope_ring_attention_f32(const float* qkv, int64_t q_batch_stride, int64_t q_time_stride, float* kv,
                                              const int64_t* offset, int32_t offset_stride, const float* freqs, float* out,
                                              int64_t o_batch_stride, int64_t o_time_stride, int32_t batch, int32_t T, int32_t H,
                                              int32_t D, int32_t cap, int32_t context, rstnet_stream_t stream) {
  RSTNET_REQUIRE(qkv && kv && offset && freqs && out, "rope_ring_attention: null pointer");
  RSTNET_REQUIRE(batch > 0 && H > 0 && cap > 0 && context > 0, "rope_ring_attention: bad shape");
  RSTNET_REQUIRE(T == 2 && D == 64 && T <= cap, "rope_ring_attention: the fused form covers streaming steps of 2 tokens at head size 64 (T=%d D=%d)", T, D);
  RSTNET_REQUIRE(((uintptr_t)qkv % 16) == 0 && ((uintptr_t)kv % 16) == 0 && ((uintptr_t)out % 16) == 0 && q_batch_stride % 4 == 0 &&
                     q_time_stride % 4 == 0 && o_batch_stride % 4 == 0 && o_time_stride % 4 == 0,
                 "rope_ring_attention: buffers and strides must be 16-byte aligned");
  const int warps = 4;
  const long long total = (long long)batch * H;
  ring_attention_pair64_kernel<<<ceil_div(total, warps), warps * 32, 0, (cudaStream_t)stream>>>(
      qkv, q_batch_stride, q_time_stride, kv, (const long long*)offset, offset_stride ? 1 : 0, out, o_batch_stride, o_time_stride, batch, T, H,
      cap, context, 0, freqs);
  count_launch();
  return check_launch("rope_ring_attention");
}

extern "C" int rstnet_ring_attention_f32(const float* qkv, int64_t q_batch_stride, int64_t q_time_stride, const float* kv,
                                         const int64_t* offset, int32_t offset_stride, float* out, int64_t o_batch_stride,
                                         int64_t o_time_stride, int32_t batch, int32_t T, int32_t H, int32_t D, int32_t cap,
                                         int32_t context, int32_t linear, rstnet_stream_t stream) {
  const int ostride = offset_stride ? 1 : 0;
  RSTNET_REQUIRE(qkv && kv && offset && out, "ring_attention: null pointer");
  RSTNET_REQUIRE(batch > 0 && T > 0 && H > 0 && D > 0 && D % 4 == 0 && D <= 128 && cap > 0 && context > 0,
                 "ring_attention: bad shape (D %% 4 == 0 and D <= 128 required)");
  const int warps = 4;
  const bool aligned16 = ((uintptr_t)qkv % 16) == 0 && ((uintptr_t)kv % 16) == 0 && ((uintptr_t)out % 16) == 0 && q_batch_stride % 4 == 0 &&
                         q_time_stride % 4 == 0 && o_batch_stride % 4 == 0 && o_time_stride % 4 == 0;
  if (T >= 2 && D == 64 && aligned16) {
    const long long total = (long long)batch * ((T + 1) / 2) * H;
    ring_attention_pair64_kernel<<<ceil_div(total, warps), warps * 32, 0, (cudaStream_t)stream>>>(
        qkv, q_batch_stride, q_time_stride, const_cast<float*>(kv), (const long long*)offset, ostride, out, o_batch_stride, o_time_stride,
        batch, T, H, cap, context, linear, nullptr);
  } else if (T >= 2) {
    const long long total = (long long)batch * ((T + 1) / 2) * H;
    ring_attention_pair_kernel<<<ceil_div(total, warps), warps * 32, warps * 2 * D * sizeof(float), (cudaStream_t)stream>>>(
        qkv, q_batch_stride, q_time_stride, kv, (const long long*)offset, ostride, out, o_batch_stride, o_time_stride, batch, T, H, D,
        cap, context, linear);
  } else {
    const long long total = (long long)batch * T * H;
    ring_attention_kernel<<<ceil_div(total, warps), warps * 32, warps * D * sizeof(float), (cudaStream_t)stream>>>(
        qkv, q_batch_stride, q_time_stride, kv, (const long long*)offset, ostride, out, o_batch_stride, o_time_stride, batch, T, H, D,
        cap, context, linear);
  }
  count_launch();
  return check_launch("ring_attention");
}
