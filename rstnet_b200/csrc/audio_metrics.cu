// Codec evaluation metrics over ragged batches of clips: the loss sums of one STFT resolution (a fused STFT-pair kernel)
// and the five moments of SI-SNR.
//
// Both kernels tile each clip on its own: CTA (b, c) covers block b of clip c, block b starting at the clip's frame (or
// sample) b * BLOCK, and writes fp64 partials to ws[c][b].  A second launch sums the partials of each clip in an order
// that depends only on the clip's length.  A clip's sums are therefore the same bytes whatever else is in the batch, where
// the clip sits in the pack and how large the pack is.  No atomics.
#include "common.cuh"
#include "../../include/rstnet_b200.h"
#include <algorithm>

namespace rstnet {

extern void count_launch();

constexpr int kStftThreads = 256;
constexpr int kStftFramesPerBlock = RSTNET_STFT_FRAMES_PER_BLOCK;
constexpr int kMomentThreads = 256;
constexpr int kMomentSamplesPerBlock = RSTNET_SISNR_SAMPLES_PER_BLOCK;
constexpr int kReduceThreads = 256;
constexpr double kMagFloor = 1e-7;   // torch.clamp(re^2 + im^2, min=1e-7) of compute_ms_stft_loss.py:21

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sum of v over the CTA in a fixed order (warp butterflies, then warp 0 over the warp totals); the result is valid in
// thread 0.  `red` holds one double per warp.
template <int NT>
__device__ __forceinline__ double block_sum_d(double v, double* red) {
  v = warp_sum_d(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();   // `red` may still be read by a previous call
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = 0.0;
  if (warp == 0) {
    t = lane < NT / 32 ? red[lane] : 0.0;
    t = warp_sum_d(t);
  }
  return t;
}

// torch.clamp semantics: NaN stays NaN (fmax would drop it)
__device__ __forceinline__ double clamp_floor(double p) { return p < kMagFloor ? kMagFloor : p; }

__device__ __forceinline__ long long reflect(long long t, long long L) {
  return t < 0 ? -t : (t >= L ? 2 * (L - 1) - t : t);
}

// One CTA: frames [b * F, min((b + 1) * F, nframes)) of clip c.  Per frame, z[n] = w[n - lpad] * (r + i d) at the reflected
// sample f * hop + n - N/2 (n inside the window's support, 0 elsewhere), loaded in bit-reversed order; log2(N) radix-2
// stages in shared memory; then R[k] = (Z[k] + conj Z[N-k]) / 2 and D[k] = (Z[k] - conj Z[N-k]) / 2i for k = 0..N/2.
// Partials: sum (T - P)^2, sum T^2, sum |log P - log T| with T = sqrt(max(|R|^2, 1e-7)), P = sqrt(max(|D|^2, 1e-7)).
__global__ void __launch_bounds__(kStftThreads) stft_pair_loss_kernel(
    const float* __restrict__ ref, const float* __restrict__ deg, const int64_t* __restrict__ offsets,
    const int64_t* __restrict__ lengths, int64_t min_len, int64_t max_len, int log2n, int hop, int win,
    const float2* __restrict__ twiddle, const float* __restrict__ window, double* __restrict__ partial, int max_blocks) {
  extern __shared__ float2 s_buf[];   // [N] data, then [N/2] twiddles
  __shared__ double s_red[kStftThreads / 32];
  const int N = 1 << log2n, half_n = N >> 1;
  float2* s_tw = s_buf + N;
  const int c = blockIdx.y, b = blockIdx.x;
  const long long L = lengths[c];
  double* out = partial + ((long long)c * max_blocks + b) * 3;
  if (L < min_len || L > max_len) {   // outside the caller's promise: the clip's sums are NaN
    if (threadIdx.x < 3) out[threadIdx.x] = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  const long long nframes = 1 + L / hop;
  const long long f0 = (long long)b * kStftFramesPerBlock;
  if (f0 >= nframes) return;
  const long long f1 = min(f0 + kStftFramesPerBlock, nframes);
  const float* r = ref + offsets[c];
  const float* d = deg + offsets[c];

  // a non-finite sample anywhere in the clip makes its sums NaN (torch.stft multiplies every sample of a frame, the
  // zeros of the padded window included); the blocks' spans [f0 * hop, f1 * hop) cover the clip
  bool bad = false;
  for (long long t = f0 * hop + threadIdx.x; t < min(f1 * hop, L); t += kStftThreads)
    bad |= !(isfinite(r[t]) && isfinite(d[t]));
  bad = __syncthreads_or(bad);
  for (int k = threadIdx.x; k < half_n; k += kStftThreads) s_tw[k] = twiddle[k];

  const int lpad = (N - win) >> 1;   // torch.stft centres the window: (n_fft - win_length) // 2 zeros on the left
  double acc_diff = 0.0, acc_true = 0.0, acc_log = 0.0;
  for (long long f = f0; f < f1; ++f) {
    __syncthreads();   // the previous frame's bins are read; twiddles are staged
    const long long t0 = f * hop - half_n;
    int differ = 0;
    for (int n = threadIdx.x; n < N; n += kStftThreads) {
      const int j = n - lpad;
      float2 z = make_float2(0.f, 0.f);
      if (j >= 0 && j < win) {
        const long long t = reflect(t0 + n, L);
        const float w = __ldg(window + j), rv = r[t], dv = d[t];
        differ |= rv != dv;
        z = make_float2(w * rv, w * dv);
      }
      s_buf[__brev(n) >> (32 - log2n)] = z;
    }
    // a frame whose two windowed inputs are equal has P == T exactly: it takes T for both (the packed FFT would leave
    // rounding differences between the two), so a signal scored against itself gives 0
    const bool same = !__syncthreads_or(differ);
    for (int s = 1; s <= log2n; ++s) {
      if (s > 1) __syncthreads();
      const int h = 1 << (s - 1);
      for (int q = threadIdx.x; q < half_n; q += kStftThreads) {
        const int j = q & (h - 1);
        const int i0 = ((q >> (s - 1)) << s) + j;
        const float2 w = s_tw[j << (log2n - s)];
        const float2 u = s_buf[i0], v = s_buf[i0 + h];
        const float2 vw = make_float2(fmaf(v.x, w.x, -v.y * w.y), fmaf(v.x, w.y, v.y * w.x));
        s_buf[i0] = make_float2(u.x + vw.x, u.y + vw.y);
        s_buf[i0 + h] = make_float2(u.x - vw.x, u.y - vw.y);
      }
    }
    __syncthreads();
    for (int k = threadIdx.x; k <= half_n; k += kStftThreads) {
      const float2 zk = s_buf[k & (N - 1)], zn = s_buf[(N - k) & (N - 1)];
      const double rr = 0.5 * ((double)zk.x + zn.x), ri = 0.5 * ((double)zk.y - zn.y);
      const double dr = 0.5 * ((double)zk.y + zn.y), di = -0.5 * ((double)zk.x - zn.x);
      const double t2 = clamp_floor(rr * rr + ri * ri), p2 = same ? t2 : clamp_floor(dr * dr + di * di);
      const double tm = sqrt(t2), pm = sqrt(p2);
      acc_diff += (tm - pm) * (tm - pm);
      acc_true += t2;
      acc_log += fabs(0.5 * (log(p2) - log(t2)));
    }
  }
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  const double s0 = block_sum_d<kStftThreads>(acc_diff, s_red);
  const double s1 = block_sum_d<kStftThreads>(acc_true, s_red);
  const double s2 = block_sum_d<kStftThreads>(acc_log, s_red);
  if (threadIdx.x == 0) {
    out[0] = bad ? nan : s0;
    out[1] = bad ? nan : s1;
    out[2] = bad ? nan : s2;
  }
}

// One CTA: samples [b * S, min((b + 1) * S, L)) of clip c -> sum r, sum d, sum r^2, sum d^2, sum r d (fp64 products of
// the fp32 samples, which are exact).
__global__ void __launch_bounds__(kMomentThreads) sisnr_moments_kernel(
    const float* __restrict__ ref, const float* __restrict__ deg, const int64_t* __restrict__ offsets,
    const int64_t* __restrict__ lengths, int64_t max_len, double* __restrict__ partial, int max_blocks) {
  __shared__ double s_red[kMomentThreads / 32];
  const int c = blockIdx.y, b = blockIdx.x;
  const long long L = lengths[c];
  double* out = partial + ((long long)c * max_blocks + b) * 5;
  if (L < 0 || L > max_len) {
    if (threadIdx.x < 5) out[threadIdx.x] = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  const long long t0 = (long long)b * kMomentSamplesPerBlock;
  if (t0 >= L) return;
  const long long t1 = min(t0 + kMomentSamplesPerBlock, L);
  const float* r = ref + offsets[c];
  const float* d = deg + offsets[c];
  double a[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (long long t = t0 + threadIdx.x; t < t1; t += kMomentThreads) {
    const double x = r[t], y = d[t];
    a[0] += x;
    a[1] += y;
    a[2] = fma(x, x, a[2]);
    a[3] = fma(y, y, a[3]);
    a[4] = fma(x, y, a[4]);
  }
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const double s = block_sum_d<kMomentThreads>(a[k], s_red);
    if (threadIdx.x == 0) out[k] = s;
  }
}

// out[c * out_stride + k] = sum over the clip's nb(c) blocks of partial[c][b][k], k < K: thread t adds blocks t, t + 256,
// ... in order, then block_sum_d.  nb(c) depends only on the clip's length.
__global__ void __launch_bounds__(kReduceThreads) reduce_partials_kernel(
    const double* __restrict__ partial, const int64_t* __restrict__ lengths, int max_blocks, int K, int per_block,
    int hop, double* __restrict__ out, long long out_stride) {
  __shared__ double s_red[kReduceThreads / 32];
  const int c = blockIdx.x;
  const long long L = lengths[c];
  // blocks the clip used: frames 1 + L / hop (STFT, hop > 0) or samples L (moments, hop == 0), per_block per block (an
  // empty clip's moments are zeros); a clip outside the caller's bounds wrote NaN to every block
  const long long items = hop > 0 ? 1 + max(L, 0LL) / hop : max(L, 0LL);
  const int nb = L < 0 ? 1 : (int)min((long long)max_blocks, (items + per_block - 1) / per_block);
  const double* p = partial + (long long)c * max_blocks * K;
  for (int k = 0; k < K; ++k) {
    double v = 0.0;
    for (int bb = threadIdx.x; bb < nb; bb += kReduceThreads) v += p[(long long)bb * K + k];
    const double s = block_sum_d<kReduceThreads>(v, s_red);
    if (threadIdx.x == 0) out[(long long)c * out_stride + k] = s;
  }
}

inline long long stft_blocks(long long max_len, int hop) {
  return (1 + max_len / hop + kStftFramesPerBlock - 1) / kStftFramesPerBlock;
}
inline long long moment_blocks(long long max_len) {
  return std::max(1LL, (max_len + kMomentSamplesPerBlock - 1) / kMomentSamplesPerBlock);
}

}  // namespace rstnet
using namespace rstnet;

extern "C" int64_t rstnet_stft_loss_workspace(int32_t clips, int64_t max_len, int32_t hop) {
  if (clips < 0 || max_len < 0 || hop < 1) return -1;
  return (int64_t)clips * stft_blocks(max_len, hop) * 3 * (int64_t)sizeof(double);
}

extern "C" int64_t rstnet_sisnr_moments_workspace(int32_t clips, int64_t max_len) {
  if (clips < 0 || max_len < 0) return -1;
  return (int64_t)clips * moment_blocks(max_len) * 5 * (int64_t)sizeof(double);
}

extern "C" int rstnet_stft_loss_sums_f32(const float* ref, const float* deg, const int64_t* offsets,
                                         const int64_t* lengths, int32_t clips, int64_t min_len, int64_t max_len,
                                         int32_t n_fft, int32_t hop, int32_t win, const float* twiddle,
                                         const float* window, double* sums, int32_t n_res, int32_t res, void* ws,
                                         int64_t ws_bytes, rstnet_stream_t stream) {
  RSTNET_REQUIRE(ref && deg && offsets && lengths && twiddle && window && sums && ws, "stft_loss: null pointer");
  RSTNET_REQUIRE(n_fft >= 64 && n_fft <= 4096 && (n_fft & (n_fft - 1)) == 0,
                 "stft_loss: n_fft must be a power of two in [64, 4096], got %d", n_fft);
  RSTNET_REQUIRE(win >= 1 && win <= n_fft, "stft_loss: win_length %d outside [1, n_fft = %d]", win, n_fft);
  RSTNET_REQUIRE(hop >= 1, "stft_loss: hop %d < 1", hop);
  RSTNET_REQUIRE(clips >= 0 && clips <= 65535, "stft_loss: %d clips outside [0, 65535]", clips);
  RSTNET_REQUIRE(n_res >= 1 && res >= 0 && res < n_res, "stft_loss: resolution %d outside [0, %d)", res, n_res);
  RSTNET_REQUIRE(min_len > n_fft / 2 && max_len >= min_len,
                 "stft_loss: clip lengths [%lld, %lld] must exceed n_fft / 2 = %d (torch.stft's reflect padding)",
                 (long long)min_len, (long long)max_len, n_fft / 2);
  const long long nb = stft_blocks(max_len, hop);
  RSTNET_REQUIRE(nb <= 0x7fffffffLL, "stft_loss: clips too long (%lld samples)", (long long)max_len);
  RSTNET_REQUIRE(ws_bytes >= rstnet_stft_loss_workspace(clips, max_len, hop),
                 "stft_loss: workspace of %lld bytes, %lld needed", (long long)ws_bytes,
                 (long long)rstnet_stft_loss_workspace(clips, max_len, hop));
  if (clips == 0) return 0;
  int log2n = 0;
  while ((1 << log2n) < n_fft) ++log2n;
  const size_t smem = (size_t)n_fft * sizeof(float2) + (size_t)(n_fft / 2) * sizeof(float2);
  static unsigned long long attr = 0;   // n_fft = 4096 fills the default 48 KB with dynamic memory alone
  smem_optin(stft_pair_loss_kernel, (4096 + 2048) * (int)sizeof(float2), attr);
  cudaStream_t st = (cudaStream_t)stream;
  double* partial = (double*)ws;
  stft_pair_loss_kernel<<<dim3((unsigned)nb, (unsigned)clips), kStftThreads, smem, st>>>(
      ref, deg, offsets, lengths, min_len, max_len, log2n, hop, win, (const float2*)twiddle, window, partial, (int)nb);
  count_launch();
  if (int rc = check_launch("stft_pair_loss")) return rc;
  reduce_partials_kernel<<<clips, kReduceThreads, 0, st>>>(partial, lengths, (int)nb, 3, kStftFramesPerBlock, hop,
                                                           sums + (long long)res * 3, (long long)n_res * 3);
  count_launch();
  return check_launch("stft_loss reduce");
}

extern "C" int rstnet_sisnr_moments_f32(const float* ref, const float* deg, const int64_t* offsets,
                                        const int64_t* lengths, int32_t clips, int64_t max_len, double* moments,
                                        void* ws, int64_t ws_bytes, rstnet_stream_t stream) {
  RSTNET_REQUIRE(ref && deg && offsets && lengths && moments && ws, "sisnr_moments: null pointer");
  RSTNET_REQUIRE(clips >= 0 && clips <= 65535, "sisnr_moments: %d clips outside [0, 65535]", clips);
  RSTNET_REQUIRE(max_len >= 0, "sisnr_moments: negative max_len");
  const long long nb = moment_blocks(max_len);
  RSTNET_REQUIRE(nb <= 0x7fffffffLL, "sisnr_moments: clips too long (%lld samples)", (long long)max_len);
  RSTNET_REQUIRE(ws_bytes >= rstnet_sisnr_moments_workspace(clips, max_len),
                 "sisnr_moments: workspace of %lld bytes, %lld needed", (long long)ws_bytes,
                 (long long)rstnet_sisnr_moments_workspace(clips, max_len));
  if (clips == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  double* partial = (double*)ws;
  sisnr_moments_kernel<<<dim3((unsigned)nb, (unsigned)clips), kMomentThreads, 0, st>>>(ref, deg, offsets, lengths,
                                                                                       max_len, partial, (int)nb);
  count_launch();
  if (int rc = check_launch("sisnr_moments")) return rc;
  reduce_partials_kernel<<<clips, kReduceThreads, 0, st>>>(partial, lengths, (int)nb, 5, kMomentSamplesPerBlock, 0,
                                                           moments, 5);
  count_launch();
  return check_launch("sisnr_moments reduce");
}
