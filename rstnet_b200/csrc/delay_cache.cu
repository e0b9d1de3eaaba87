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

// ---- the prompt of a row (LMGen.prefill_streams): P steps of cache_in / cache_out in one launch, the sampled tokens
// given.  One CTA per listed row, one thread per codebook; each thread walks its codebook's ring through the P steps in
// shared memory, in the order the two kernels above run them, so every column, the feed and the final offset equal P
// pairs of launches on an active row.  The row list travels in the launch's parameters, so a captured launch keeps it.
struct DelayPromptRows {
  int row[RSTNET_DELAY_PROMPT_MAX_ROWS];
  int start[RSTNET_DELAY_PROMPT_MAX_ROWS];
  int len[RSTNET_DELAY_PROMPT_MAX_ROWS];
};

__global__ void __launch_bounds__(kDelayCacheThreads) delay_cache_prompt_kernel(
    long long* __restrict__ cache, long long* __restrict__ off, long long* __restrict__ valid,
    const long long* __restrict__ delays, const long long* __restrict__ prompt, int prompt_stride, long long* __restrict__ feed,
    int feed_stride, const DelayPromptRows rows, int K, int dep_q, int CT, int max_delay, long long text_init,
    long long audio_init) {
  extern __shared__ long long rings[];   // [K][CT]
  const int k = threadIdx.x;
  const int b = rows.row[blockIdx.x];
  const int P = rows.len[blockIdx.x];
  const long long s0 = rows.start[blockIdx.x];
  const long long o0 = off[b];
  long long* ring = rings + k * CT;
  long long* g = cache + ((long long)b * K + k) * CT;
  for (int c = 0; c < CT; ++c) ring[c] = g[c];
  const long long d = delays[k];
  const long long init = k == 0 ? text_init : audio_init;
#pragma unroll 4
  for (int t = 0; t < P; ++t) {
    const long long o = o0 + t;
    const long long tok = prompt[(s0 + t) * prompt_stride + k];
    if (k > dep_q) ring[mod_ct(o + d, CT)] = tok;                  // cache_in: the user token
    if (o <= d) ring[mod_ct(o, CT)] = init;                        // cache_in: the initial token
    feed[(s0 + t) * feed_stride + k] = ring[mod_ct(o, CT)];         // cache_in: the temporal transformer's input
    if (k <= dep_q) ring[mod_ct(o + 1, CT)] = tok;                 // cache_out: the sampled token
  }
  for (int c = 0; c < CT; ++c) g[c] = ring[c];
  __syncthreads();   // every thread of the row has read off[b]
  if (k == 0) {
    off[b] = o0 + P;
    valid[b] = (o0 + P > max_delay) ? 1 : 0;
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

extern "C" int rstnet_lm_delay_cache_prompt(int64_t* cache, int64_t* off, int64_t* valid, const int64_t* delays,
                                            const int64_t* prompt, int32_t prompt_stride, int64_t* feed, int32_t feed_stride,
                                            const int32_t* rows, const int32_t* starts, const int32_t* lengths, int32_t n, int32_t B,
                                            int32_t K, int32_t dep_q, int32_t CT, int32_t max_delay, int64_t text_init,
                                            int64_t audio_init, rstnet_stream_t stream) {
  RSTNET_REQUIRE(cache && off && valid && delays && prompt && feed && rows && starts && lengths,
                 "lm_delay_cache_prompt: null pointer");
  RSTNET_REQUIRE(n >= 0 && n <= RSTNET_DELAY_PROMPT_MAX_ROWS, "lm_delay_cache_prompt: %d rows (at most %d)", n,
                 RSTNET_DELAY_PROMPT_MAX_ROWS);
  RSTNET_REQUIRE(B > 0 && K >= 1 && K <= kDelayCacheThreads && dep_q >= 0 && dep_q < K && max_delay >= 0 &&
                 CT == max_delay + 2 && (long long)K * CT * 8 <= 48 * 1024,
                 "lm_delay_cache_prompt: bad shape (B=%d, K=%d, dep_q=%d, CT=%d, max_delay=%d)", B, K, dep_q, CT, max_delay);
  RSTNET_REQUIRE(prompt_stride >= K && feed_stride >= K, "lm_delay_cache_prompt: row strides too small");
  DelayPromptRows list;
  int m = 0;
  for (int i = 0; i < n; ++i) {
    RSTNET_REQUIRE(rows[i] >= 0 && rows[i] < B, "lm_delay_cache_prompt: row %d outside [0, %d)", rows[i], B);
    RSTNET_REQUIRE(lengths[i] >= 0 && starts[i] >= 0, "lm_delay_cache_prompt: row %d has a negative start or length", rows[i]);
    for (int j = 0; j < i; ++j)
      RSTNET_REQUIRE(rows[j] != rows[i], "lm_delay_cache_prompt: row %d listed twice", rows[i]);
    if (lengths[i] == 0) continue;   // left untouched
    list.row[m] = rows[i];
    list.start[m] = starts[i];
    list.len[m] = lengths[i];
    ++m;
  }
  if (m == 0) return 0;
  delay_cache_prompt_kernel<<<dim3(m), dim3(K), (size_t)K * CT * sizeof(long long), (cudaStream_t)stream>>>(
      (long long*)cache, (long long*)off, (long long*)valid, (const long long*)delays, (const long long*)prompt, prompt_stride,
      (long long*)feed, feed_stride, list, K, dep_q, CT, max_delay, (long long)text_init, (long long)audio_init);
  count_launch();
  return check_launch("lm_delay_cache_prompt");
}
