// The acoustic-delay token cache of LMGen.step (models/model.py:490-562; moshi/models/lm.py LMGen.step), one ring of
// CT = max_delay + 2 columns per stream and codebook, with a per-stream offset so that streams of one batch can start,
// and be held, independently.  Two small kernels around the LM frame, both graph-capturable:
//
//   cache_in  (before the temporal step), active rows only:
//     cache[b, k, (off + delays[k]) % CT] = user[b, k - dep_q - 1]         k = dep_q + 1 .. K - 1
//     cache[b, k, off % CT] = initial[k]          if off <= delays[k]      (text_init for k = 0, audio_init otherwise)
//   then, every row:  seq[b, k] = cache[b, k, off % CT]   (a held row feeds ids < -1 as the zero token -1: its step is
//   discarded, and a column it has not yet written may still hold the ungenerated id -2)
//
//   cache_out (after the last depth sample), active rows only:
//     cache[b, k, (off + 1) % CT] = tokens[b, k]                            k = 0 .. dep_q
//     off += 1
//     out[b, k] = cache[b, k, (off - max_delay + delays[k]) mod CT]         k = 0 .. dep_q
//     valid[b] = off > max_delay
//
// A held row's cache, offset, valid flag and output row are not written.  One thread per (row, codebook): every
// cache entry a thread reads or writes lies in its own codebook's ring, so threads only share the row's offset, which
// cache_out advances after the whole row has read it.
#include "common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {

extern void count_launch();

constexpr int kDelayCacheThreads = 128;

__device__ __forceinline__ long long mod_ct(long long x, int CT) {
  const long long r = x % CT;
  return r < 0 ? r + CT : r;
}

__global__ void __launch_bounds__(kDelayCacheThreads) delay_cache_in_kernel(
    long long* __restrict__ cache, const long long* __restrict__ off, const long long* __restrict__ active,
    const long long* __restrict__ delays, const long long* __restrict__ user, int user_stride, long long* __restrict__ seq,
    int seq_stride, int B, int K, int dep_q, int CT, long long text_init, long long audio_init) {
  const int k = threadIdx.x;
  const int b = blockIdx.x * blockDim.y + threadIdx.y;
  if (b >= B || k >= K) return;
  const long long o = off[b];
  long long* ring = cache + ((long long)b * K + k) * CT;
  const bool act = active == nullptr || active[b] != 0;
  if (act) {
    const long long d = delays[k];
    if (k > dep_q) ring[mod_ct(o + d, CT)] = user[(long long)b * user_stride + (k - dep_q - 1)];
    if (o <= d) ring[mod_ct(o, CT)] = k == 0 ? text_init : audio_init;
  }
  const long long v = ring[mod_ct(o, CT)];
  seq[(long long)b * seq_stride + k] = (!act && v < -1) ? -1 : v;
}

__global__ void __launch_bounds__(kDelayCacheThreads) delay_cache_out_kernel(
    long long* __restrict__ cache, long long* __restrict__ off, const long long* __restrict__ active,
    const long long* __restrict__ delays, const long long* __restrict__ tokens, int tok_stride, long long* __restrict__ out,
    int out_stride, long long* __restrict__ valid, int B, int K, int dep_q, int CT, int max_delay) {
  const int k = threadIdx.x;
  const int b = blockIdx.x * blockDim.y + threadIdx.y;
  const bool row = b < B;
  const bool act = row && (active == nullptr || active[b] != 0);
  const long long o = row ? off[b] : 0;
  if (act && k <= dep_q) {
    long long* ring = cache + ((long long)b * K + k) * CT;
    ring[mod_ct(o + 1, CT)] = tokens[(long long)b * tok_stride + k];
    out[(long long)b * out_stride + k] = ring[mod_ct(o + 1 - max_delay + delays[k], CT)];
  }
  __syncthreads();   // every thread of the row has read off[b]
  if (act && k == 0) {
    off[b] = o + 1;
    valid[b] = (o + 1 > max_delay) ? 1 : 0;
  }
}

// (row, codebook) threads: x = codebook, y = rows of the CTA
inline void delay_cache_grid(int B, int K, dim3& grid, dim3& block) {
  const int rows = kDelayCacheThreads / K;
  block = dim3(K, rows);
  grid = dim3((B + rows - 1) / rows);
}

}  // namespace rstnet
using namespace rstnet;

extern "C" int rstnet_lm_delay_cache_in(int64_t* cache, const int64_t* off, const int64_t* active, const int64_t* delays,
                                        const int64_t* user, int32_t user_stride, int64_t* seq, int32_t seq_stride, int32_t B,
                                        int32_t K, int32_t dep_q, int32_t CT, int64_t text_init, int64_t audio_init,
                                        rstnet_stream_t stream) {
  RSTNET_REQUIRE(cache && off && delays && user && seq, "lm_delay_cache_in: null pointer");
  RSTNET_REQUIRE(B > 0 && K >= 1 && K <= kDelayCacheThreads && dep_q >= 0 && dep_q < K && CT >= 2,
                 "lm_delay_cache_in: bad shape (B=%d, K=%d, dep_q=%d, CT=%d)", B, K, dep_q, CT);
  RSTNET_REQUIRE(user_stride >= K - dep_q - 1 && seq_stride >= K, "lm_delay_cache_in: row strides too small");
  dim3 grid, block;
  delay_cache_grid(B, K, grid, block);
  delay_cache_in_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(
      (long long*)cache, (const long long*)off, (const long long*)active, (const long long*)delays, (const long long*)user,
      user_stride, (long long*)seq, seq_stride, B, K, dep_q, CT, (long long)text_init, (long long)audio_init);
  count_launch();
  return check_launch("lm_delay_cache_in");
}

extern "C" int rstnet_lm_delay_cache_out(int64_t* cache, int64_t* off, const int64_t* active, const int64_t* delays,
                                         const int64_t* tokens, int32_t tok_stride, int64_t* out, int32_t out_stride,
                                         int64_t* valid, int32_t B, int32_t K, int32_t dep_q, int32_t CT, int32_t max_delay,
                                         rstnet_stream_t stream) {
  RSTNET_REQUIRE(cache && off && delays && tokens && out && valid, "lm_delay_cache_out: null pointer");
  RSTNET_REQUIRE(B > 0 && K >= 1 && K <= kDelayCacheThreads && dep_q >= 0 && dep_q < K && max_delay >= 0 &&
                 CT == max_delay + 2, "lm_delay_cache_out: bad shape (B=%d, K=%d, dep_q=%d, CT=%d, max_delay=%d)", B, K,
                 dep_q, CT, max_delay);
  RSTNET_REQUIRE(tok_stride >= dep_q + 1 && out_stride >= dep_q + 1, "lm_delay_cache_out: row strides too small");
  dim3 grid, block;
  delay_cache_grid(B, K, grid, block);
  delay_cache_out_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(
      (long long*)cache, (long long*)off, (const long long*)active, (const long long*)delays, (const long long*)tokens,
      tok_stride, (long long*)out, out_stride, (long long*)valid, B, K, dep_q, CT, max_delay);
  count_launch();
  return check_launch("lm_delay_cache_out");
}
