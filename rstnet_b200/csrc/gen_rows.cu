// Per-row generation window of the batch generation loop (infer.py `_TTSRows`), advanced on the device after the last
// depth sample of every frame, inside the frame's CUDA graph.  The reference loop (MLLM_v2/infer_no_streaming.py:229-292)
// decides two things per generated frame from the frame's own tokens and the utterance's window:
//
//   the early stop (:284-286):  g_idx > minlen and some codebook l in 3..7 has a token >= 2048: the frame is dropped and
//                               the utterance ends (codebook 0, the semantic one, is not read; ported as written);
//   the candidate sets (:264-283) of the NEXT frame g' = g_idx + 1:  codebook l samples from 2049 ids when l > 0 and
//                               pre_gen_len + g' > minlen, from 2048 otherwise (all 2049 on frame 0, which the host sets).
//
// One thread per row.  A row's record is rec[b] = {pre_gen_len, minlen, maxlen, g_idx, mode}; mode & 3 is HELD (the row
// is not generating: nothing is written but its status), FIXED (no stop rule: a TTS row of known length) or WINDOWED,
// and mode & RSTNET_GEN_ARGMAX gives the row the whole card (the argmax path has no candidate masks, sampling.py:107-154;
// the stop rule still applies, as in the reference with use_sampling False).  The frame just generated is g_idx:
//   status[b] = STOPPED  (windowed, stop rule)      -> mode becomes HELD
//             = LAST     (g_idx + 1 >= maxlen)      -> mode becomes HELD
//             = RUNNING  otherwise: g_idx += 1 and row_valid[b] = the next frame's counts
//             = IDLE     for a held row (no frame of it is generated, or it already ended)
#include "common.cuh"
#include "../../include/rstnet_b200.h"

namespace rstnet {
extern void count_launch();
}

namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) gen_rows_advance_kernel(const long long* __restrict__ tokens, int tok_stride,
                                                                     int* __restrict__ rec, int* __restrict__ row_valid,
                                                                     int valid_stride, int* __restrict__ status, int B,
                                                                     int dep_q, int card) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int* r = rec + (long long)b * RSTNET_GEN_REC;
  const int mode = r[4], kind = mode & 3;
  if (kind != RSTNET_GEN_FIXED && kind != RSTNET_GEN_WINDOWED) {
    status[b] = RSTNET_GEN_IDLE;
    return;
  }
  const int pre = r[0], minlen = r[1], maxlen = r[2], g = r[3];
  const long long* t = tokens + (long long)b * tok_stride + 1;   // audio codebooks 0 .. dep_q - 1
  bool stop = false;
  if (kind == RSTNET_GEN_WINDOWED && g > minlen)
    for (int l = 3; l < dep_q && l <= 7; ++l) stop |= t[l] >= 2048;
  if (stop || g + 1 >= maxlen) {
    status[b] = stop ? RSTNET_GEN_STOPPED : RSTNET_GEN_LAST;
    r[4] = mode & ~3;                                             // HELD, keeping the argmax flag
    return;
  }
  const int gn = g + 1;
  r[3] = gn;
  status[b] = RSTNET_GEN_RUNNING;
  const bool argmax = (mode & RSTNET_GEN_ARGMAX) != 0;
  // pre + gn > minlen without overflow for any int window
  const bool open = (long long)pre + gn > (long long)minlen;
  int* v = row_valid + (long long)b * valid_stride;
  for (int l = 0; l < dep_q; ++l) v[l] = argmax ? card : ((l > 0 && open) ? 2049 : 2048);
}

}  // namespace

extern "C" int rstnet_lm_gen_rows_advance(const int64_t* tokens, int32_t tok_stride, int32_t* rec, int32_t* row_valid,
                                          int32_t valid_stride, int32_t* status, int32_t B, int32_t dep_q, int32_t card,
                                          rstnet_stream_t stream) {
  RSTNET_REQUIRE(tokens && rec && row_valid && status, "lm_gen_rows_advance: null pointer");
  RSTNET_REQUIRE(B > 0 && dep_q >= 1 && card >= 2049, "lm_gen_rows_advance: bad shape (B=%d, dep_q=%d, card=%d)", B, dep_q,
                 card);
  RSTNET_REQUIRE(tok_stride >= dep_q + 1 && valid_stride >= dep_q,
                 "lm_gen_rows_advance: row strides too small (tok_stride=%d, valid_stride=%d, dep_q=%d)", tok_stride,
                 valid_stride, dep_q);
  gen_rows_advance_kernel<<<(B + kThreads - 1) / kThreads, kThreads, 0, (cudaStream_t)stream>>>(
      (const long long*)tokens, tok_stride, rec, row_valid, valid_stride, status, B, dep_q, card);
  rstnet::count_launch();
  return rstnet::check_launch("lm_gen_rows_advance");
}
