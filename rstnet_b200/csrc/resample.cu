// Polyphase sinc resampling (torchaudio.transforms.Resample with its defaults), fp32.
//
//   out[r, q] (q = j*n + p < out_len) = sum_{i < S} xv(r, j*o + x_shift + start[p] + i) * taps[p][i]
//   xv(r, t) = x[r*x_row_stride + t] if 0 <= t < x_len, else 0
//
// taps [n][S] is the table trimmed to each phase's run of nonzero taps (zero-padded at the end), start[p] the run's
// first tap.  The sum starts at +0.0f and accumulates with fmaf in increasing i whatever the tiling: the batch form
// (x_shift = -w) and the streaming form (x = carry buffer, x_shift = 0) are the same compiled body with another origin,
// which is what makes them bit-identical.
#include "common.cuh"
#include "../../include/rstnet_b200.h"
#include <algorithm>

namespace rstnet {

extern void count_launch();

constexpr int kResampleThreads = 256;
constexpr int kResampleMaxTableBytes = RSTNET_RESAMPLE_MAX_TABLE_BYTES;
constexpr int kResampleSmemBudget = 200 * 1024;

// One CTA: JT consecutive blocks (JT*n outputs) of one row at a time, looping over rows.  The trimmed table (row stride
// Sp = S | 1, so that neighbouring phases fall in different banks) and the CTA's input span live in shared memory; the
// span is staged with coalesced, bounds-checked loads (the zero padding of the batch form), the outputs are written by
// consecutive threads to consecutive q.
__global__ void __launch_bounds__(kResampleThreads) resample_poly_kernel(
    const float* __restrict__ x, long long x_row_stride, long long x_len, long long x_shift, const float* __restrict__ taps,
    const int* __restrict__ start, int n, int o, int S, int start_max, float* __restrict__ out, long long out_row_stride,
    long long out_len, int rows, int JT) {
  extern __shared__ float smem[];
  const int Sp = S | 1;
  float* s_taps = smem;
  int* s_start = reinterpret_cast<int*>(smem + (size_t)n * Sp);
  float* s_x = reinterpret_cast<float*>(s_start + n);
  const int span = (JT - 1) * o + start_max + S;
  for (int i = threadIdx.x; i < n * S; i += blockDim.x) s_taps[(i / S) * Sp + i % S] = taps[i];
  for (int p = threadIdx.x; p < n; p += blockDim.x) s_start[p] = start[p];

  const long long j0 = (long long)blockIdx.x * JT;
  const long long q0 = j0 * n;
  const int nq = (int)min((long long)JT * n, out_len - q0);
  const long long base = j0 * o + x_shift;
  for (int r = blockIdx.y; r < rows; r += gridDim.y) {
    const float* xr = x + (long long)r * x_row_stride;
    __syncthreads();   // the previous row's span is no longer read (and, first time round, the table is staged)
    for (int i = threadIdx.x; i < span; i += blockDim.x) {
      const long long t = base + i;
      s_x[i] = (t >= 0 && t < x_len) ? xr[t] : 0.f;
    }
    __syncthreads();
    float* orow = out + (long long)r * out_row_stride + q0;
    for (int lq = threadIdx.x; lq < nq; lq += blockDim.x) {
      const int jl = lq / n, p = lq - jl * n;
      const int s0 = s_start[p];
      float acc = 0.f;
      if (s0 < 0 || s0 > start_max) {
        acc = __int_as_float(0x7fffffff);   // a start outside [0, start_max] breaks the caller's promise: poison
      } else {
        const float* xs = s_x + jl * o + s0;
        const float* hs = s_taps + p * Sp;
#pragma unroll 4
        for (int i = 0; i < S; ++i) acc = fmaf(xs[i], hs[i], acc);
      }
      orow[lq] = acc;
    }
  }
}

}  // namespace rstnet
using namespace rstnet;

extern "C" int rstnet_resample_f32(const float* x, int64_t x_row_stride, int64_t x_len, int64_t x_shift, const float* taps,
                                   const int32_t* start, int32_t n, int32_t o, int32_t S, int32_t start_max, float* out,
                                   int64_t out_row_stride, int64_t out_len, int32_t rows, rstnet_stream_t stream) {
  RSTNET_REQUIRE(x && taps && start && out, "resample: null pointer");
  RSTNET_REQUIRE(n >= 1 && o >= 1 && S >= 1 && start_max >= 0, "resample: bad table shape (n=%d, o=%d, S=%d, start_max=%d)",
                 n, o, S, start_max);
  RSTNET_REQUIRE((long long)n * S * 4 <= kResampleMaxTableBytes,
                 "resample: the trimmed table [%d phases x %d taps] is %lld bytes, above the %d-byte cap", n, S,
                 (long long)n * S * 4, kResampleMaxTableBytes);
  RSTNET_REQUIRE(rows >= 0 && x_len >= 0 && out_len >= 0, "resample: negative size");
  RSTNET_REQUIRE(rows <= 1 || out_row_stride >= out_len, "resample: output rows overlap (stride %lld < out_len %lld)",
                 (long long)out_row_stride, (long long)out_len);
  if (rows == 0 || out_len == 0) return 0;
  // blocks per CTA: about 2048 outputs (or one table's worth, when the table is larger), capped by the span's share of
  // shared memory
  const long long table_bytes = ((long long)n * (S | 1) + n) * 4;
  const long long span_budget = (kResampleSmemBudget - table_bytes) / 4 - start_max - S;
  RSTNET_REQUIRE(span_budget >= 0, "resample: start_max %d does not fit in shared memory", start_max);
  long long jt = (std::max(2048LL, (long long)n * S) + n - 1) / n;
  jt = std::min(jt, 1 + span_budget / o);
  const long long blocks = (out_len + n - 1) / n;
  jt = std::max(1LL, std::min(jt, blocks));
  const long long grid_x = (blocks + jt - 1) / jt;
  RSTNET_REQUIRE(grid_x <= 0x7fffffffLL, "resample: output too long (%lld samples)", (long long)out_len);
  const size_t smem = (size_t)table_bytes + (size_t)((jt - 1) * o + start_max + S) * 4;
  static unsigned long long attr = 0;
  smem_optin(resample_poly_kernel, kResampleSmemBudget, attr);
  const dim3 grid((unsigned)grid_x, (unsigned)std::min(rows, 65535));
  resample_poly_kernel<<<grid, kResampleThreads, smem, (cudaStream_t)stream>>>(
      x, x_row_stride, x_len, x_shift, taps, (const int*)start, n, o, S, start_max, out, out_row_stride, out_len, rows, (int)jt);
  count_launch();
  return check_launch("resample");
}
