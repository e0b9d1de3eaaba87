// Small HBM-bound kernels of the Mimi codec: the two degenerate convs (Cin==1, Cout==1), the
// depthwise upsampling transposed conv, padding / streaming-carry row moves, LayerNorm.
#include "common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {
extern void count_launch();

// ---------------------------------------------------------------- conv Cin == 1
// block = (Cout threads in x) x (TT time steps in y-loop); x window staged in smem.
template <int TT>
__global__ void conv_cin1_kernel(const float* __restrict__ x, long long xbs, long long xts, const float* __restrict__ w,
                                 const float* __restrict__ bias, float* __restrict__ out, float* __restrict__ out2,
                                 long long obs, long long ots, int T, int Cout, int k, int post_act, int act2) {
  extern __shared__ float xs[];  // TT + k - 1
  const int b = blockIdx.y;
  const long long t0 = (long long)blockIdx.x * TT;
  const int nthreads = blockDim.x;
  const float* xb = x + (long long)b * xbs;
  const int nwin = min((long long)TT, (long long)T - t0) + k - 1;
  for (int i = threadIdx.x; i < nwin; i += nthreads) xs[i] = xb[(t0 + i) * xts];
  __syncthreads();
  for (int co = threadIdx.x; co < Cout; co += nthreads) {
    float wr[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) wr[j] = j < k ? w[co * k + j] : 0.f;
    const float bv = bias ? bias[co] : 0.f;
    const int tn = (int)min((long long)TT, (long long)T - t0);
    for (int t = 0; t < tn; ++t) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (j < k) acc = fmaf(xs[t + j], wr[j], acc);
      acc += bv;
      // out2 exists only for the tensor-core plans (pre-activated copy for the next conv): same ex2-based ELU as their epilogues
      if (out2) out2[(long long)b * obs + (t0 + t) * ots + co] = act2 == ACT_ELU ? elu_fast(acc) : apply_act(acc, act2);
      out[(long long)b * obs + (t0 + t) * ots + co] = apply_act(acc, post_act);
    }
  }
}

// ---------------------------------------------------------------- conv Cout == 1
// one warp per 32 consecutive outputs; rows staged in smem padded to Cin+1 floats.
__global__ void conv_cout1_kernel(const float* __restrict__ x, long long xbs, long long xts, const float* __restrict__ w,
                                  const float* __restrict__ bias, float* __restrict__ out, long long obs,
                                  int T, int Cin, int k) {
  extern __shared__ float sm[];
  const int warps = blockDim.x / 32;
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int K = k * Cin;
  float* ws = sm;                                             // K weights
  float* xs = sm + K + warp * (32 + k - 1) * (Cin + 1);       // per-warp rows
  for (int i = threadIdx.x; i < K; i += blockDim.x) ws[i] = w[i];
  const int b = blockIdx.y;
  const long long t0 = ((long long)blockIdx.x * warps + warp) * 32;
  const float* xb = x + (long long)b * xbs;
  const int nrows = (int)min(32LL, (long long)T - t0) + k - 1;
  if (t0 < T) {
    const int total = nrows * Cin;
    if ((Cin & 3) == 0 && (xts & 3) == 0 && ((uintptr_t)xb & 15) == 0) {
      // 16-byte loads, four row pieces per lane in flight: the kernel is a pure stream over the input (126 MB per 256-stream
      // frame at 24 kHz) and scalar loads left it far below HBM bandwidth
      const int c4n = Cin >> 2, total4 = nrows * c4n;
      for (int i0 = lane; i0 < total4; i0 += 128) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = i0 + 32 * u;
          if (i < total4) v[u] = __ldg(reinterpret_cast<const float4*>(xb + (t0 + i / c4n) * xts) + (i % c4n));
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = i0 + 32 * u;
          if (i < total4) {
            float* d = xs + (i / c4n) * (Cin + 1) + 4 * (i % c4n);
            d[0] = v[u].x; d[1] = v[u].y; d[2] = v[u].z; d[3] = v[u].w;
          }
        }
      }
    } else if ((Cin & (Cin - 1)) == 0) {   // power-of-two channel count: shift / mask instead of a division per element
      const int sh = 31 - __clz(Cin);
      for (int i = lane; i < total; i += 32) {
        const int r = i >> sh, c = i & (Cin - 1);
        xs[r * (Cin + 1) + c] = xb[(t0 + r) * xts + c];
      }
    } else {
      for (int i = lane; i < total; i += 32) {
        int r = i / Cin, c = i % Cin;
        xs[r * (Cin + 1) + c] = xb[(t0 + r) * xts + c];
      }
    }
  }
  __syncthreads();
  if (t0 >= T) return;
  const long long t = t0 + lane;
  if (t < T) {
    float acc = 0.f;
    for (int j = 0; j < k; ++j) {
      const float* xr = xs + (lane + j) * (Cin + 1);
      const float* wr = ws + j * Cin;
      int c = 0;
      if ((Cin & 3) == 0 && ((j * Cin) & 3) == 0) {
        for (; c < Cin; c += 4) {   // weights as one broadcast 128-bit read per four taps; same accumulation order
          const float4 w4 = *reinterpret_cast<const float4*>(wr + c);
          acc = fmaf(xr[c], w4.x, acc); acc = fmaf(xr[c + 1], w4.y, acc);
          acc = fmaf(xr[c + 2], w4.z, acc); acc = fmaf(xr[c + 3], w4.w, acc);
        }
      }
      for (; c < Cin; ++c) acc = fmaf(xr[c], wr[c], acc);
    }
    out[(long long)b * obs + t] = acc + (bias ? bias[0] : 0.f);
  }
}

// ---------------------------------------------------------------- depthwise transposed conv, k = 2*stride
__global__ void convtr_depthwise_kernel(const float* __restrict__ x, long long xbs, long long xts,
                                        const float* __restrict__ w, float* __restrict__ out, long long obs,
                                        long long ots, int T, int C, int s) {
  const long long total = (long long)T * s * C;
  const int b = blockIdx.y;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long tau = i / C;
    const long long t = tau / s;
    const int j = (int)(tau % s);
    const float* xb = x + (long long)b * xbs;
    const float cur = xb[(t + 1) * xts + c], prev = xb[t * xts + c];  // row 0 is the carry row x[-1]
    // same association as the reference: contribution of x[t-1] (tap j+s) was accumulated first
    // (`partial`), then x[t]'s tap j is added (streaming.py:287-292)
    out[(long long)b * obs + tau * ots + c] = fmaf(cur, w[c * 2 * s + j], prev * w[c * 2 * s + j + s]);
  }
}

// ---------------------------------------------------------------- row fill / carry copy
// only_if_zero: per-stream counters when oz_stride == 1 (stream of column c in batch b = b * (C / cps) + c / cps,
// cps = channels per stream: the batch-major layout has C == cps, the time-major one C == B * cps), one shared counter
// when oz_stride == 0.
__global__ void rows_fill_kernel(float* __restrict__ buf, long long bs, int C, int row0, int nrows, int mode,
                                 int src_row, const long long* __restrict__ only_if_zero, int oz_stride, int cps) {
  if (only_if_zero && !oz_stride && *only_if_zero != 0) return;
  const int b = blockIdx.y;
  float* bb = buf + (long long)b * bs;
  const long long total = (long long)nrows * C;
  const int spb = C / cps;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    if (only_if_zero && oz_stride && only_if_zero[(long long)b * spb + c / cps] != 0) continue;
    bb[(long long)row0 * C + i] = mode == 1 ? bb[(long long)src_row * C + c] : 0.f;
  }
}

// Each thread owns one channel column and moves its rows in ascending order, so a carry that is
// longer than the chunk (src and dst row ranges overlap, src_row >= dst_row) still shifts correctly.
// active (optional): one flag per stream; a stream whose flag is 0 keeps its carry rows (a frame scheduler "holds" the
// rows that had no input this tick: their state must not advance).  Stream of column c of batch b =
// b * (C / cps) + c / cps with cps = the entry's channels per stream (0 -> C).
__global__ void rows_copy_table_kernel(const rstnet_row_copy* __restrict__ table, int n_entries,
                                       const long long* __restrict__ active) {
  const int e = blockIdx.y, b = blockIdx.z;
  if (e >= n_entries) return;
  const rstnet_row_copy ent = table[e];
  float* bb = ent.buf + (long long)b * ent.batch_stride;
  const float* src = bb + (long long)ent.src_row * ent.C;
  float* dst = bb + (long long)ent.dst_row * ent.C;
  const int cps = ent.cps > 0 ? ent.cps : ent.C;
  const int spb = ent.C / cps;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < ent.C; c += gridDim.x * blockDim.x) {
    if (active && active[(long long)b * spb + c / cps] == 0) continue;
    for (int r = 0; r < ent.nrows; ++r) dst[(long long)r * ent.C + c] = src[(long long)r * ent.C + c];
  }
}

__global__ void counter_add_kernel(long long* c, long long d, int n, const long long* __restrict__ active) {
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (!active || active[i] != 0) c[i] += d;
}

// ---------------------------------------------------------------- LayerNorm: one warp per row
__global__ void layer_norm_kernel(const float* __restrict__ x, long long xbs, const float* __restrict__ w,
                                  const float* __restrict__ bias, float* __restrict__ y, long long rows, int rows_per_batch,
                                  int dim, float eps) {
  const long long row = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (row >= rows) return;
  const float* xr = x + (row / rows_per_batch) * xbs + (row % rows_per_batch) * dim;
  float s = 0.f;
  for (int i = lane; i < dim; i += 32) s += xr[i];
  const float mean = warp_sum(s) / (float)dim;
  float v = 0.f;
  for (int i = lane; i < dim; i += 32) { const float d = xr[i] - mean; v = fmaf(d, d, v); }
  const float var = warp_sum(v) / (float)dim;
  const float rstd = 1.0f / sqrtf(var + eps);
  float* yr = y + row * dim;
  for (int i = lane; i < dim; i += 32) yr[i] = (xr[i] - mean) * rstd * w[i] + bias[i];
}

// Same arithmetic, but the row lives in registers: ONE pass over memory instead of three dependent ones (the 25 Hz
// transformer launches this 32 times per frame on 512 rows: the three-pass form ran at memory latency).
template <int NPL>
__global__ void layer_norm_reg_kernel(const float* __restrict__ x, long long xbs, const float* __restrict__ w,
                                      const float* __restrict__ bias, float* __restrict__ y, long long rows, int rows_per_batch,
                                      int dim, float eps) {
  const long long row = (long long)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
  const int lane = threadIdx.x % 32;
  if (row >= rows) return;
  const float* xr = x + (row / rows_per_batch) * xbs + (row % rows_per_batch) * dim;
  float v[NPL];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NPL; ++i) v[i] = xr[lane + 32 * i];
#pragma unroll
  for (int i = 0; i < NPL; ++i) s += v[i];
  const float mean = warp_sum(s) / (float)dim;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NPL; ++i) { const float d = v[i] - mean; q = fmaf(d, d, q); }
  const float var = warp_sum(q) / (float)dim;
  const float rstd = 1.0f / sqrtf(var + eps);
  float* yr = y + row * dim;
#pragma unroll
  for (int i = 0; i < NPL; ++i) yr[lane + 32 * i] = (v[i] - mean) * rstd * w[lane + 32 * i] + bias[lane + 32 * i];
}

}  // namespace rstnet
using namespace rstnet;

extern "C" int rstnet_conv1d_cin1_f32(const float* x, int64_t xbs, int64_t xts, const float* w, const float* bias, float* out,
                                      float* out2, int64_t obs, int64_t ots, int32_t batch, int32_t T, int32_t Cout,
                                      int32_t k, int32_t post_act, int32_t act2, rstnet_stream_t stream) {
  RSTNET_REQUIRE(x && w && out, "conv1d_cin1: null pointer");
  RSTNET_REQUIRE(batch > 0 && T > 0 && Cout > 0 && k > 0 && k <= 16, "conv1d_cin1: bad shape (k<=16 required, k=%d)", k);
  constexpr int TT = 128;
  dim3 grid((unsigned)ceil_div(T, TT), (unsigned)batch);
  const int threads = Cout >= 128 ? 128 : (Cout >= 64 ? 64 : 32);
  conv_cin1_kernel<TT><<<grid, threads, (TT + k - 1) * sizeof(float), (cudaStream_t)stream>>>(
      x, xbs, xts, w, bias, out, out2, obs, ots, T, Cout, k, post_act, act2);
  count_launch();
  return check_launch("conv1d_cin1");
}

extern "C" int rstnet_conv1d_cout1_f32(const float* x, int64_t xbs, int64_t xts, const float* w, const float* bias,
                                       float* out, int64_t obs, int32_t batch, int32_t T, int32_t Cin, int32_t k,
                                       rstnet_stream_t stream) {
  RSTNET_REQUIRE(x && w && out, "conv1d_cout1: null pointer");
  RSTNET_REQUIRE(batch > 0 && T > 0 && Cin > 0 && k > 0, "conv1d_cout1: bad shape");
  const int warps = 4;
  const size_t smem = ((size_t)k * Cin + (size_t)warps * (32 + k - 1) * (Cin + 1)) * sizeof(float);
  RSTNET_REQUIRE(smem <= 200 * 1024, "conv1d_cout1: Cin*k too large for shared memory");
  static unsigned long long attr = 0;
  smem_optin(conv_cout1_kernel, 200 * 1024, attr);
  dim3 grid((unsigned)ceil_div(T, 32 * warps), (unsigned)batch);
  conv_cout1_kernel<<<grid, warps * 32, smem, (cudaStream_t)stream>>>(x, xbs, xts, w, bias, out, obs, T, Cin, k);
  count_launch();
  return check_launch("conv1d_cout1");
}

extern "C" int rstnet_convtr1d_depthwise_f32(const float* x, int64_t xbs, int64_t xts, const float* w, float* out,
                                             int64_t obs, int64_t ots, int32_t batch, int32_t T, int32_t C,
                                             int32_t stride, rstnet_stream_t stream) {
  RSTNET_REQUIRE(x && w && out, "convtr1d_depthwise: null pointer");
  RSTNET_REQUIRE(batch > 0 && T > 0 && C > 0 && stride > 0, "convtr1d_depthwise: bad shape");
  const long long total = (long long)T * stride * C;
  int gx = ceil_div(total, 256);
  if (gx > 4096) gx = 4096;
  convtr_depthwise_kernel<<<dim3(gx, batch), 256, 0, (cudaStream_t)stream>>>(x, xbs, xts, w, out, obs, ots, T, C, stride);
  count_launch();
  return check_launch("convtr1d_depthwise");
}

extern "C" int rstnet_rows_fill_f32(float* buf, int64_t bs, int32_t batch, int32_t C, int32_t row0, int32_t nrows,
                                    int32_t mode, int32_t src_row, const int64_t* only_if_zero, int32_t only_if_zero_stride,
                                    int32_t channels_per_stream, rstnet_stream_t stream) {
  RSTNET_REQUIRE(buf, "rows_fill: null pointer");
  if (channels_per_stream <= 0) channels_per_stream = C;
  RSTNET_REQUIRE(C % channels_per_stream == 0, "rows_fill: C (%d) must be a multiple of channels_per_stream (%d)", C, channels_per_stream);
  if (nrows <= 0 || batch <= 0) return 0;
  const long long total = (long long)nrows * C;
  int gx = ceil_div(total, 256);
  if (gx > 1024) gx = 1024;
  rows_fill_kernel<<<dim3(gx, batch), 256, 0, (cudaStream_t)stream>>>(buf, bs, C, row0, nrows, mode, src_row,
                                                                     (const long long*)only_if_zero, only_if_zero_stride ? 1 : 0,
                                                                     channels_per_stream);
  count_launch();
  return check_launch("rows_fill");
}

extern "C" int rstnet_rows_copy_table_f32(const rstnet_row_copy* table_dev, int32_t n_entries, int32_t batch,
                                          const int64_t* active, rstnet_stream_t stream) {
  RSTNET_REQUIRE(table_dev, "rows_copy_table: null pointer");
  if (n_entries <= 0 || batch <= 0) return 0;
  RSTNET_REQUIRE(n_entries <= 65535 && batch <= 65535, "rows_copy_table: too many entries / batch");
  // grid.x strides over the channel columns of an entry (up to batch*C in the time-major layout)
  rows_copy_table_kernel<<<dim3(batch > 1 ? 4 : 256, n_entries, batch), 256, 0, (cudaStream_t)stream>>>(table_dev, n_entries,
                                                                                                          (const long long*)active);
  count_launch();
  return check_launch("rows_copy_table");
}

extern "C" int rstnet_counter_add(int64_t* counter, int64_t delta, int32_t n, const int64_t* active, rstnet_stream_t stream) {
  RSTNET_REQUIRE(counter && n >= 1, "counter_add: bad argument");
  counter_add_kernel<<<1, n >= 256 ? 256 : 32, 0, (cudaStream_t)stream>>>((long long*)counter, delta, n, (const long long*)active);
  count_launch();
  return check_launch("counter_add");
}

extern "C" int rstnet_layer_norm_f32(const float* x, int64_t x_batch_stride, const float* weight, const float* bias,
                                     float* y, int32_t batch, int32_t rows_per_batch, int32_t dim, float eps,
                                     rstnet_stream_t stream) {
  RSTNET_REQUIRE(x && weight && bias && y, "layer_norm: null pointer");
  const long long rows = (long long)batch * rows_per_batch;
  if (rows <= 0) return 0;
  if (dim == 512 || dim == 256 || dim == 1024) {
    const int w4 = 4;
    const dim3 grid((unsigned)ceil_div(rows, w4));
    cudaStream_t st = (cudaStream_t)stream;
    if (dim == 512) layer_norm_reg_kernel<16><<<grid, w4 * 32, 0, st>>>(x, x_batch_stride, weight, bias, y, rows, rows_per_batch, dim, eps);
    else if (dim == 256) layer_norm_reg_kernel<8><<<grid, w4 * 32, 0, st>>>(x, x_batch_stride, weight, bias, y, rows, rows_per_batch, dim, eps);
    else layer_norm_reg_kernel<32><<<grid, w4 * 32, 0, st>>>(x, x_batch_stride, weight, bias, y, rows, rows_per_batch, dim, eps);
    count_launch();
    return check_launch("layer_norm");
  }
  const int warps = 8;
  layer_norm_kernel<<<ceil_div(rows, warps), warps * 32, 0, (cudaStream_t)stream>>>(x, x_batch_stride, weight, bias, y,
                                                                                 rows, rows_per_batch, dim, eps);
  count_launch();
  return check_launch("layer_norm");
}
