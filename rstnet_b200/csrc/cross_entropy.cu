// Cross-entropy and accuracy over bf16 logit rows: the F.cross_entropy(..., reduction='none') / argmax / mask sums of
// CrossEntropyAndAccuracy (models/model.py:31-65), for the teacher-forced scoring of a sequence.
//
// Launch 1 (`ce_rows_kernel<NT>`): NT threads per row (a warp for the 2 050-wide audio rows, a 512-thread CTA for the
// 152 064-wide text rows), one pass over the row.  Each thread keeps an online (max m, t = sum of exp(x - m) over the
// elements seen except one element equal to m) pair in fp32 and the first maximum; 8-element vectors are summed locally
// before they join the running sum, which keeps the fp32 summation error of a 152 064-wide row near 1e-7.  Loss =
// (m - x[label]) + log1p(t): exact difference of two bf16 values plus a log1p, so a confident row keeps its relative
// precision.  Rows are read with 16-byte loads from the first 16-byte boundary on (scalar head and tail), so any row
// stride works.
// Launch 2 (`ce_reduce_kernel`): one CTA per accumulator entry (slot, group) sums its rows in a fixed order in fp64 and
// adds the result to the caller's accumulator: no atomics, identical bytes for identical calls.
#include <cuda_bf16.h>
#include <climits>

#include "common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {
extern void count_launch();
typedef __nv_bfloat16 bf16;

// Sticky error word of this file (bit 0: label outside [0, V) that is not the ignore id), read by
// rstnet_device_error_flags together with the other kernels' words.
__device__ unsigned int g_ce_dev_err = 0;
unsigned int ce_read_errors(bool clear) {
  unsigned int v = 0;
  cudaMemcpyFromSymbol(&v, g_ce_dev_err, sizeof(v));
  if (clear && v) { const unsigned int z = 0; cudaMemcpyToSymbol(g_ce_dev_err, &z, sizeof(z)); }
  return v;
}

namespace {

constexpr float NEG_INF = -__builtin_huge_valf();

struct CeState {
  float m;    // running max over non-NaN elements (NaN counts as -inf here; a NaN anywhere poisons the loss below)
  float t;    // sum of exp(x - m) over the elements seen, except one element equal to m
  float bv;   // first maximum: value and index (INT_MAX: none yet)
  int bi;
  int nan_i;  // first NaN index (INT_MAX: none)
};

__device__ __forceinline__ void ce_merge(CeState& a, const CeState& b) {
  if (b.m > a.m) {
    a.t = b.t + (a.t + 1.f) * expf(a.m - b.m);
    a.m = b.m;
  } else if (b.m < a.m) {
    a.t += (b.t + 1.f) * expf(b.m - a.m);
  } else {
    a.t += b.t + 1.f;   // equal maxima (two empty states only meet when the row max is -inf: NaN loss below)
  }
  if (b.bv > a.bv || (b.bv == a.bv && b.bi < a.bi)) { a.bv = b.bv; a.bi = b.bi; }
  a.nan_i = min(a.nan_i, b.nan_i);
}

__device__ __forceinline__ CeState ce_shfl(const CeState& s, int o) {
  CeState r;
  r.m = __shfl_xor_sync(0xffffffffu, s.m, o);
  r.t = __shfl_xor_sync(0xffffffffu, s.t, o);
  r.bv = __shfl_xor_sync(0xffffffffu, s.bv, o);
  r.bi = __shfl_xor_sync(0xffffffffu, s.bi, o);
  r.nan_i = __shfl_xor_sync(0xffffffffu, s.nan_i, o);
  return r;
}

// N consecutive elements with indices i0.. (increasing across the calls of one thread).  A NaN is recorded (first index)
// and then takes no part in the sums or the maximum.
template <int N>
__device__ __forceinline__ void ce_chunk(CeState& s, float (&x)[N], int i0) {
  int fk = -1;
#pragma unroll
  for (int k = N - 1; k >= 0; --k)
    if (x[k] != x[k]) { fk = k; x[k] = NEG_INF; }
  if (fk >= 0 && s.nan_i == INT_MAX) s.nan_i = i0 + fk;
  float cm = x[0];
#pragma unroll
  for (int k = 1; k < N; ++k) cm = fmaxf(cm, x[k]);
  bool skip = false;
  if (cm > s.m) {
    s.t = (s.t + 1.f) * expf(s.m - cm);
    s.m = cm;
    skip = true;   // the first element equal to the new max is the one t leaves out
  }
  if (cm > s.bv) {
    int k0 = 0;
#pragma unroll
    for (int k = N - 1; k >= 0; --k)
      if (x[k] == cm) k0 = k;
    s.bv = cm;
    s.bi = i0 + k0;
  }
  float ls = 0.f;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    float e = x[k] == s.m ? 1.f : expf(x[k] - s.m);   // (x == m also covers -inf == -inf)
    if (skip && x[k] == s.m) { e = 0.f; skip = false; }
    ls += e;
  }
  s.t += ls;
}

__device__ __forceinline__ void unpack8(const uint4& v, float (&x)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = __bfloat1622float2(h[j]);
    x[2 * j] = f.x;
    x[2 * j + 1] = f.y;
  }
}

}  // namespace

// NT threads per row (NT == 32: ROWS_PER_CTA rows of one warp each; NT > 32: one row per CTA).
template <int NT>
__global__ void __launch_bounds__(NT >= 256 ? NT : 256)
ce_rows_kernel(const bf16* __restrict__ logits, long long row_stride, int rows, int V, int groups,
               const long long* __restrict__ labels, const long long* __restrict__ ignore_ids,
               const int* __restrict__ row_slot, float* __restrict__ nll, int* __restrict__ pred) {
  constexpr int RPC = NT >= 256 ? 1 : 256 / NT;
  const int lane = threadIdx.x % NT;
  const int row = blockIdx.x * RPC + threadIdx.x / NT;
  if (row >= rows) return;   // (NT < 256: whole groups of NT threads leave together; NT >= 256: RPC == 1)
  if (row_slot && row_slot[row] < 0) {   // padding row of a scoring chunk: not read
    if (lane == 0) { nll[row] = 0.f; pred[row] = -1; }
    return;
  }
  const bf16* x = logits + (long long)row * row_stride;
  // elements before the first 16-byte boundary, then 8-element vectors, then the tail
  const int mis = (int)((reinterpret_cast<uintptr_t>(x) >> 1) & 7);
  const int head = min(V, mis ? 8 - mis : 0);
  const int nvec = (V - head) >> 3;
  const int tail0 = head + nvec * 8;
  CeState s{NEG_INF, 0.f, NEG_INF, INT_MAX, INT_MAX};
  if (lane < head) {
    float v[1] = {__bfloat162float(x[lane])};
    ce_chunk<1>(s, v, lane);
  }
  const uint4* xv = reinterpret_cast<const uint4*>(x + head);
  constexpr int U = 4;   // 16-byte loads in flight per thread
  int j = lane;
  for (; j + (U - 1) * NT < nvec; j += U * NT) {
    uint4 r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) r[u] = __ldg(xv + j + u * NT);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float v[8];
      unpack8(r[u], v);
      ce_chunk<8>(s, v, head + 8 * (j + u * NT));
    }
  }
  for (; j < nvec; j += NT) {
    float v[8];
    unpack8(__ldg(xv + j), v);
    ce_chunk<8>(s, v, head + 8 * j);
  }
  for (int i = tail0 + lane; i < V; i += NT) {   // < 8 elements
    float v[1] = {__bfloat162float(x[i])};
    ce_chunk<1>(s, v, i);
  }
  // fixed-shape tree: lanes of a warp, then (NT > 32) the warps of the CTA
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const CeState r = ce_shfl(s, o);
    ce_merge(s, r);
  }
  if (NT > 32) {
    __shared__ CeState part[NT / 32 > 1 ? NT / 32 : 1];
    const int w = threadIdx.x / 32;
    if ((threadIdx.x & 31) == 0) part[w] = s;
    __syncthreads();
    if (threadIdx.x != 0) return;
    s = part[0];
    for (int i = 1; i < NT / 32; ++i) ce_merge(s, part[i]);
  } else if (lane != 0) {
    return;
  }
  const int g = row % groups;
  const long long y = labels[row];
  const bool ignored = ignore_ids && y == ignore_ids[g];
  float loss;
  if (ignored) {
    loss = 0.f;
  } else if (y < 0 || y >= V) {
    atomicOr(&g_ce_dev_err, 1u);   // where F.cross_entropy raises: NaN row + error bit 0
    loss = __int_as_float(0x7fc00000);
  } else if (s.nan_i != INT_MAX || s.m == NEG_INF) {
    loss = __int_as_float(0x7fc00000);   // as log_softmax: a NaN logit, or a row without a finite maximum
  } else {
    loss = (s.m - __bfloat162float(x[y])) + log1pf(s.t);
  }
  nll[row] = loss;
  // torch.argmax: a NaN is the maximum; ties go to the first index (a row of -inf only: index 0)
  pred[row] = s.nan_i != INT_MAX ? s.nan_i : (s.bi == INT_MAX ? 0 : s.bi);
}

// acc[(slot * groups + g) * 5 + {0..4}] += (sum w*nll, #(w != 0), #(w == 1), #correct(w != 0), #correct(w == 1)) over
// the rows r with r % groups == g and slot(r) == slot, in increasing row order per thread and a fixed tree.
__global__ void __launch_bounds__(256)
ce_reduce_kernel(const float* __restrict__ nll, const int* __restrict__ pred, const long long* __restrict__ labels,
                 const float* __restrict__ w, const int* __restrict__ row_slot, int rows, int groups, double* __restrict__ acc) {
  const int e = blockIdx.x;
  const int slot = e / groups, g = e % groups;
  double a[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int r = g + groups * (int)threadIdx.x; r < rows; r += groups * (int)blockDim.x) {
    if (row_slot ? row_slot[r] != slot : slot != 0) continue;
    const float wr = w[r];
    const bool ok = (long long)pred[r] == labels[r];
    a[0] += (double)wr * (double)nll[r];
    a[1] += wr != 0.f ? 1.0 : 0.0;
    a[2] += wr == 1.f ? 1.0 : 0.0;
    a[3] += (ok && wr != 0.f) ? 1.0 : 0.0;
    a[4] += (ok && wr == 1.f) ? 1.0 : 0.0;
  }
  __shared__ double sh[5][256];
#pragma unroll
  for (int k = 0; k < 5; ++k) sh[k][threadIdx.x] = a[k];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) {
#pragma unroll
      for (int k = 0; k < 5; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x < 5) acc[(long long)e * 5 + threadIdx.x] += sh[threadIdx.x][0];
}

}  // namespace rstnet
using namespace rstnet;

extern "C" int rstnet_lm_cross_entropy_bf16(const void* logits, int64_t row_stride, int32_t rows, int32_t V, int32_t groups,
                                            const int64_t* labels, const int64_t* ignore_ids, const float* weights,
                                            const int32_t* row_slot, int32_t n_slots, float* nll, int32_t* pred, double* acc,
                                            rstnet_stream_t stream) {
  RSTNET_REQUIRE(logits && labels && weights && nll && pred && acc, "lm_cross_entropy: null pointer");
  RSTNET_REQUIRE(rows > 0 && V > 0 && groups > 0 && row_stride >= V, "lm_cross_entropy: bad shape (rows %d, V %d, groups %d, "
                 "row_stride %lld)", rows, V, groups, (long long)row_stride);
  RSTNET_REQUIRE(n_slots > 0 && (row_slot || n_slots == 1), "lm_cross_entropy: n_slots %d without a row_slot map", n_slots);
  RSTNET_REQUIRE((reinterpret_cast<uintptr_t>(logits) & 1) == 0, "lm_cross_entropy: logits not 2-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* lg = (const bf16*)logits;
  const long long* lb = (const long long*)labels;
  const long long* ig = (const long long*)ignore_ids;
  if (V > 8192) {
    ce_rows_kernel<512><<<rows, 512, 0, st>>>(lg, (long long)row_stride, rows, V, groups, lb, ig, row_slot, nll, pred);
  } else {
    ce_rows_kernel<32><<<ceil_div(rows, 8), 256, 0, st>>>(lg, (long long)row_stride, rows, V, groups, lb, ig, row_slot, nll, pred);
  }
  count_launch();
  if (int rc = check_launch("lm_cross_entropy rows")) return rc;
  ce_reduce_kernel<<<n_slots * groups, 256, 0, st>>>(nll, pred, lb, weights, row_slot, rows, groups, acc);
  count_launch();
  return check_launch("lm_cross_entropy reduce");
}
