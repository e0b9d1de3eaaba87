/* rstnet_b200 — C ABI of the H100 (sm_90a) kernels behind RSTnet's real-time inference hot path.
 *
 * The reference (yangdongchao/RSTnet) is pure Python/PyTorch and has no FFI of its own; the
 * drop-in boundary is its Python class surface (SURVEY.md §8b).  Each entry point below replaces
 * the ATen call cluster of one reference method (cited as file:line of the reference repository) and is
 * what a replacement library must export.  Conventions:
 *   - plain C: raw DEVICE pointers, explicit sizes/strides in ELEMENTS, no torch types;
 *   - the caller owns every buffer (activations, KV rings, conv carry rows, scratch);
 *   - `stream` is a cudaStream_t (torch.cuda.current_stream().cuda_stream); launches are
 *     asynchronous, never synchronise the device, and are CUDA-graph capturable;
 *   - return 0 on success, non-zero on error with text in rstnet_last_error() (thread-local);
 *     functions never throw and never call exit();
 *   - no CPU fallback: without a CUDA device every compute entry point fails.
 *
 * Activation layout is time-major / channels-last ("NWC"): [B, T, C] fp32 with C contiguous.
 * A causal conv over that layout is a GEMM whose A rows are OVERLAPPING windows of the input
 * (row (b,t) = k*Cin contiguous floats starting at input row t*stride), so convs, transposed
 * convs and linears all go through rstnet_gemm_rows_f32.
 */
#ifndef RSTNET_B200_H
#define RSTNET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* rstnet_stream_t; /* cudaStream_t */

enum { RSTNET_ACT_NONE = 0, RSTNET_ACT_ELU = 1, RSTNET_ACT_GELU = 2 };

int rstnet_version(void);
const char* rstnet_last_error(void);
/* number of kernels this library has launched in this process (bench.py's gpu_launches) */
int64_t rstnet_launch_count(void);
/* Sticky device-side error bits of the CURRENT device (the call synchronises it; clear != 0 resets them).
 * Kernels cannot raise, so where the reference's ATen call would (nn.Embedding / F.embedding with an id outside the
 * table, llama_streaming.py:505-517, core_vq.py:198-206; cos.index_select beyond block_size, llama_streaming.py:972-975)
 * the kernel poisons its output row with NaN (or clamps, for RVQ codes) and sets: bit 0 (1) id / code out of range,
 * bit 1 (2) RoPE position beyond the cos/sin tables. */
uint32_t rstnet_device_error_flags(int clear);

/* ---- strided-row GEMM: C[b,t,:] = post( R[b,t,:] + scale * (pre(A_row(b,t)) . Wt + bias) )
 * A_row(b,t) = K contiguous floats at A + b*a_batch_stride + t*a_row_stride.
 * Wt is [K][N] row-major.  bias/scale/R may be NULL.  Requires K%4==0, N%4==0, 16-byte aligned
 * rows.  Replaces: nn.Conv1d inside StreamingConv1d.forward (modules/conv.py:232-254,
 * modules/streaming.py:216-244); nn.ConvTranspose1d inside StreamingConvTranspose1d.forward
 * (conv.py:306-329, streaming.py:270-303; k == 2*stride rewritten as a GEMM over [x[t-1],x[t]]);
 * F.linear in StreamingMultiheadAttention / StreamingTransformerLayer
 * (modules/transformer.py:375-419, 550-577); the 1x1 Conv1d projections of
 * ResidualVectorQuantizer (quantization/vq.py:80-91); ELU / GELU / LayerScale / residual adds
 * around them (modules/seanet.py:92-94, transformer.py:559-577). */
typedef struct {
  const float* A;
  int64_t a_batch_stride, a_row_stride;
  const float* Wt;
  const float* bias;
  const float* scale;
  const float* R;
  int64_t r_batch_stride, r_row_stride;
  float* C;
  int64_t c_batch_stride, c_row_stride;
  int32_t batch, rows, N, K;
  int32_t pre_act, post_act;
  /* taps > 1: K = taps * kc and tap j of a row starts at A_row + j*tap_stride (a causal conv over the time-major
   * [T, B, C] layout, where consecutive time steps are B*C elements apart); taps <= 1: K contiguous. */
  int32_t taps;
  int64_t tap_stride;
} rstnet_gemm_rows_args;
int rstnet_gemm_rows_f32(const rstnet_gemm_rows_args* args, rstnet_stream_t stream);

/* ---- the same contraction on the tensor cores (warpgroup MMA, wgmma, with operands staged by TMA), as a plan bound
 * to fixed buffers (the library owns only the TMA descriptors and
 * tile configuration; the caller owns all tensors):
 *   D[(i,o), n] = sum_tap sum_c A[c, i + tap*tap_di, o*o_mul + tap*tap_do] * W[n, tap*Kc + c]
 * A is the activation buffer viewed as a 3-D tensor (c, i, o) with element strides
 * (1, a_i_stride, a_o_stride); W is [N][taps*Kc] (K contiguous).  Output element (i, o, n) goes to
 * C + o*c_o_stride + i*c_i_stride + n, or, when n_split > 0 (transposed conv: n = j*n_split + co),
 * to C + o*c_o_stride + i*c_i_stride + j*c_split_stride + co; R (optional residual) likewise.
 * Epilogue: post(R + scale*(acc + bias)); pre_act (RSTNET_ACT_NONE or RSTNET_ACT_ELU; others are rejected by
 * rstnet_tc_gemm_create) is applied to A in registers as the operand fragments are built.
 * precision 0 = 3xTF32 split (fp32-equivalent, for RVQ-index exactness; W must already be rounded to
 * TF32 and W_lo = tf32(w - W) supplied -- see rstnet_tf32_split_f32), 1 = single TF32 pass.
 * The kernel is persistent (at most one CTA per SM walking the 128 x 32 or 128 x 64 output tiles, or 64-row tiles in
 * K-pair mode, below).  ELU, as pre- and
 * post-activation, is evaluated with ex2.approx.
 * Same reference call sites as rstnet_gemm_rows_f32. */
typedef struct rstnet_tc_plan rstnet_tc_plan;
typedef struct {
  const float* A;
  int64_t a_i_stride, a_o_stride;
  int32_t a_c_extent, a_i_extent, a_o_extent;
  int32_t taps, tap_di, tap_do, o_mul;
  const float* W;
  const float* W_lo;
  int32_t N, Kc;
  int32_t I_out, O_out;
  float* C;
  int64_t c_i_stride, c_o_stride, c_split_stride;
  const float* R;
  int64_t r_i_stride, r_o_stride, r_split_stride;
  const float* bias;
  const float* scale;
  int32_t n_split;
  int32_t pre_act, post_act, precision;
  float* C2;    /* optional second output act2(R + scale*(acc + bias)) written with C's strides */
  int32_t act2;
} rstnet_tc_gemm_desc;
int rstnet_tc_gemm_create(const rstnet_tc_gemm_desc* desc, rstnet_tc_plan** out);
int rstnet_tc_gemm_run(const rstnet_tc_plan* plan, rstnet_stream_t stream);
void rstnet_tc_gemm_destroy(rstnet_tc_plan* plan);
/* the plan's tile grid: 128-row M tiles (I tiles x O_out), N tiles, tile width */
int rstnet_tc_gemm_grid(const rstnet_tc_plan* plan, int32_t* grid_x, int32_t* grid_y, int32_t* tile_n);
/* K-pair mode: 64-row tiles whose promotion chunks (K = 128) alternate between the CTA's two consumer warpgroups, one
 * warpgroup adding the other's chunk sums in chunk order, so the output is bit-identical to the 128-row form.
 * rstnet_tc_gemm_create picks it for the few-tile, long-K launches: when the 128-row tiles fit in one round of the
 * SMs (tiles128 <= SMs) and
 *   ceil(tiles64 / SMs) * ceil(chunks / 2) * 4  <  taps * Kc / 32
 * (rounds times serial K stages per tile); a tie keeps 128-row tiles.  rstnet_tc_gemm_create_ex takes the choice explicitly:
 * kpair = -1 (the same rule), 0 (128-row tiles) or 1 (K-pair).  rstnet_tc_gemm_kpair reports the plan's mode. */
int rstnet_tc_gemm_create_ex(const rstnet_tc_gemm_desc* desc, int32_t kpair, rstnet_tc_plan** out);
int rstnet_tc_gemm_kpair(const rstnet_tc_plan* plan, int32_t* on);
/* ---- one SEANet residual block (modules/seanet.py SEANetResnetBlock, kernel 3, compress 2) of C = 64 or 128 channels
 * on the tensor cores, as one plan and one launch:
 *   h[i, t] = ELU(b1 + sum_{tap<3} W1[:, tap*C:(tap+1)*C] ELU(y[i, t - 2 + tap]))        (C -> C/2)
 *   out[i, t] = ELU(y[i, t] + b2 + W2 h[i, t])                                              (C/2 -> C, + skip)
 * the block plus the ELU that follows it in the encoder and decoder.  Element c of stream i at row `row` of the raw
 * input is Y[row*y_o_stride + i*y_i_stride + c]; rows 0 and 1 are the causal context of output step 0, so output step t
 * reads rows t, t + 1, t + 2 and y_rows >= O_out + 2.  Output element (i, t, c) goes to
 * out + t*out_o_stride + i*out_i_stride + c.  Precision 0 only (3xTF32): W1 / W1_lo are the TF32 split of
 * the k3 weights [C/2][3C] (K = tap-major, channel-minor), W2 / W2_lo of the 1x1 weights [C][C/2] (rstnet_tf32_split_f32).
 * The result is bit-identical to the two rstnet_tc_gemm launches (k3 with pre_act = post_act = ELU into a hidden
 * buffer, then 1x1 with R = y and post_act = ELU); the hidden tensor stays in shared memory and y is read once. */
typedef struct rstnet_tc_resblock_plan rstnet_tc_resblock_plan;
typedef struct {
  const float* Y;
  int64_t y_i_stride, y_o_stride;
  int32_t channels;
  int32_t I_out, O_out, y_rows;
  const float* W1;
  const float* W1_lo;
  const float* b1;
  const float* W2;
  const float* W2_lo;
  const float* b2;
  float* out;
  int64_t out_i_stride, out_o_stride;
} rstnet_tc_resblock_desc;
int rstnet_tc_resblock_create(const rstnet_tc_resblock_desc* desc, rstnet_tc_resblock_plan** out);
int rstnet_tc_resblock_run(const rstnet_tc_resblock_plan* plan, rstnet_stream_t stream);
void rstnet_tc_resblock_destroy(rstnet_tc_resblock_plan* plan);

/* hi[i] = tf32_rna(x[i]); lo[i] = tf32_rna(x[i] - hi[i])  (one-time weight preparation for precision 0)
 * tf32_rna rounds to nearest with ties away from zero.  Non-finite x: NaN -> hi a quiet NaN (a NaN in the top 19 bits, the
 * ones the tensor core reads), lo = 0; +-Inf -> hi = +-Inf, lo = 0.  Finite x with |x| >= 0x7F7FF000 (about 3.4e38)
 * rounds to hi = +-Inf and lo = -+Inf: keep weights and activations below that.
 * Non-finite activations: a NaN or +-Inf in A (after pre_act) gives the non-finite outputs the float64 contraction gives,
 * with the same class, at both precisions.  An infinite WEIGHT at precision 0 gives a non-finite output where the float64
 * result is +-Inf, but it may be NaN: the split product adds a_lo * w_hi = a_lo * Inf, which is NaN where a_lo == 0 and
 * opposes a_hi * Inf where a_lo has the other sign. */
int rstnet_tf32_split_f32(const float* x, float* hi, float* lo, int64_t n, rstnet_stream_t stream);

/* ---- first SEANet encoder conv, Cin == 1 (modules/seanet.py:177-187): sample (b, t) at
 * x + b*x_batch_stride + t*x_time_stride (padded, T + k - 1 samples per stream), w [Cout][k],
 * out rows at out + b*out_batch_stride + t*out_time_stride. */
int rstnet_conv1d_cin1_f32(const float* x, int64_t x_batch_stride, int64_t x_time_stride, const float* w, const float* bias,
                           float* out, float* out2 /* optional act2 copy, same strides */, int64_t out_batch_stride,
                           int64_t out_time_stride, int32_t batch, int32_t T, int32_t Cout, int32_t k,
                           int32_t post_act, int32_t act2, rstnet_stream_t stream);

/* ---- last SEANet decoder conv, Cout == 1 (modules/seanet.py:372-384): x row (b, t) =
 * Cin floats at x + b*x_batch_stride + t*x_time_stride (padded, already activated),
 * w [k*Cin] ((tap, ci) order), out [B, T]. */
int rstnet_conv1d_cout1_f32(const float* x, int64_t x_batch_stride, int64_t x_time_stride, const float* w,
                            const float* bias, float* out, int64_t out_batch_stride, int32_t batch,
                            int32_t T, int32_t Cin, int32_t k, rstnet_stream_t stream);

/* ---- ConvTrUpsample1d, depthwise ConvTranspose1d k == 2*stride, no bias
 * (modules/resample.py:86-119): x [B, 1+T, C] with one carry row in front, w [C][k],
 * out[b, t*s+j, c] = x[t]*w[c][j] + x[t-1]*w[c][j+s]. */
int rstnet_convtr1d_depthwise_f32(const float* x, int64_t x_batch_stride, int64_t x_time_stride,
                                  const float* w, float* out, int64_t out_batch_stride,
                                  int64_t out_time_stride, int32_t batch, int32_t T, int32_t C,
                                  int32_t stride, rstnet_stream_t stream);

/* ---- row utilities for padding / streaming carry (F.pad in conv.py:81-100;
 * `previous` / `partial` state in streaming.py:216-303).
 * fill: rows [row0,row0+nrows) of buf[B, *, C] := 0 (mode 0) or := row `src_row` (mode 1, replicate).
 * If `only_if_zero` is non-NULL the fill happens only when *only_if_zero == 0 (first streaming
 * step).  copy_table: executes a device-resident table of row-block copies (all conv carries of
 * one step in a single launch); entry layout = rstnet_row_copy. */
int rstnet_rows_fill_f32(float* buf, int64_t batch_stride, int32_t batch, int32_t C, int32_t row0,
                         int32_t nrows, int32_t mode, int32_t src_row, const int64_t* only_if_zero,
                         int32_t only_if_zero_stride /* 0: one shared counter; 1: one per stream, stream of column c of
                         batch b = b*(C/channels_per_stream) + c/channels_per_stream */,
                         int32_t channels_per_stream, rstnet_stream_t stream);
/* fill_tail: the right padding a non-streaming StreamingConv1d applies at the end of a clip (modules/conv.py:245-254: zeros
 * for the SEANet convs, replicate for ConvDownsample1d), applied inside a streaming chunk whose clip ends there.  Stream s
 * (numbered as in rows_fill) keeps rows [row0, row0 + n_s) with n_s = min(nrows, ceil(valid[s] / valid_div)); rows
 * [row0 + n_s, row0 + nrows) := 0 (mode 0) or := row row0 + n_s - 1 (mode 1, needs row0 >= 1).  valid: device int64
 * [streams] (samples of the clip in this chunk; valid_div = the layer's total stride, so n_s is the layer's ceil-chain
 * length), read at run time: one captured launch serves every step, and a stream with n_s == nrows is left alone. */
int rstnet_rows_fill_tail_f32(float* buf, int64_t batch_stride, int32_t batch, int32_t C, int32_t row0, int32_t nrows,
                              int32_t mode, const int64_t* valid, int64_t valid_div, int32_t channels_per_stream,
                              rstnet_stream_t stream);
typedef struct {
  float* buf;
  int64_t batch_stride; /* elements */
  int32_t C, src_row, dst_row, nrows;
  int32_t cps;          /* channels per stream within a row of C columns (0 -> C): which `active` flag governs a column */
  int32_t reserved;
} rstnet_row_copy;
/* active (optional, device int64 [streams]): a stream whose flag is 0 keeps its carry rows -- the frame scheduler's
 * "hold" for batch rows that received no input this tick (their state must not advance). */
int rstnet_rows_copy_table_f32(const rstnet_row_copy* table_dev, int32_t n_entries, int32_t batch,
                               const int64_t* active, rstnet_stream_t stream);
/* counter[i] += delta for i < n (device int64 counters: StreamingTransformer.offset, transformer.py:686-690; one per
 * stream so that a single stream can be reset / admitted while the others keep running) */
int rstnet_counter_add(int64_t* counter, int64_t delta, int32_t n, const int64_t* active /* optional, [n]: 0 = hold */,
                       rstnet_stream_t stream);
/* counter[i] += delta[i] for i < n (delta [n] int64 on the device): positions of a ragged prefill chunk. */
int rstnet_counter_add_rows(int64_t* counter, const int64_t* delta, int32_t n, rstnet_stream_t stream);

/* ---- nn.LayerNorm over the last dim, eps inside sqrt (modules/transformer.py:113-114).
 * x row (b,t) at x + b*x_batch_stride + t*dim; y is contiguous [batch*rows_per_batch, dim]. */
int rstnet_layer_norm_f32(const float* x, int64_t x_batch_stride, const float* weight, const float* bias,
                          float* y, int32_t batch, int32_t rows_per_batch, int32_t dim, float eps,
                          rstnet_stream_t stream);

/* ---- codec transformer attention (modules/transformer.py:375-419, modules/rope.py:11-68,
 * RingKVCache transformer.py:211-278).
 * qkv row (b,t) = 3*H*D floats laid out (p h d) at qkv + b*q_batch_stride + t*q_time_stride.  Step 1 rotates q,k by the pair-RoPE angle of absolute
 * position (*offset + t), writes rotated q back in place and k,v into the ring kv[2][B][H][cap][D]
 * at slot (pos % cap).  Step 2 attends each query over keys with positions in
 * (pos_q - context, pos_q] that are still in the ring, fp32 softmax, out [B, T, H*D].
 * `offset` is a device int64 (positions already written before this call): one shared counter (offset_stride 0) or
 * one per stream, offset[b] (offset_stride 1; streams admitted or reset at different times).  linear != 0: kv is a
 * plain [0, cap) buffer holding every position (non-streaming, KVCacheResult.from_kv); linear == 0:
 * ring semantics of RingKVCache.complete, including its quirk that the oldest slot (position
 * end - cap) is labelled `end_offset` and therefore masked once the ring has wrapped. */
int rstnet_rope_kv_append_f32(float* qkv, int64_t q_batch_stride, int64_t q_time_stride, float* kv,
                              const int64_t* offset, int32_t offset_stride, const float* freqs, int32_t batch,
                              int32_t T, int32_t H, int32_t D, int32_t cap, rstnet_stream_t stream);
int rstnet_ring_attention_f32(const float* qkv, int64_t q_batch_stride, int64_t q_time_stride,
                              const float* kv, const int64_t* offset, int32_t offset_stride, float* out,
                              int64_t o_batch_stride, int64_t o_time_stride, int32_t batch, int32_t T,
                              int32_t H, int32_t D, int32_t cap, int32_t context, int32_t linear,
                              rstnet_stream_t stream);
/* Both steps in one launch for a streaming step of T = 2 tokens at D = 64 (the 25 Hz codec transformers): the warp
 * that owns (stream, head) rotates q in registers, rotates / appends k, v itself and then attends (ring semantics, same
 * arithmetic as the two calls above; qkv is left untouched). */
int rstnet_rope_ring_attention_f32(const float* qkv, int64_t q_batch_stride, int64_t q_time_stride, float* kv,
                                   const int64_t* offset, int32_t offset_stride, const float* freqs, float* out,
                                   int64_t o_batch_stride, int64_t o_time_stride, int32_t batch, int32_t T, int32_t H,
                                   int32_t D, int32_t cap, int32_t context, rstnet_stream_t stream);

/* ---- SplitResidualVectorQuantizer.encode (quantization/vq.py:305-315; core_vq.py:179-185,
 * 365-376): x [N, ldx] holds the two projected latents (rvq_first at column 0, rvq_rest at
 * column dim); Et [n_q][dim][bins] are the centroids TRANSPOSED, enorm [n_q][bins] their squared
 * norms.  Distances follow torch.cdist's matmul form sqrt(max(|x|^2+|e|^2-2x.e, 0)); argmin
 * keeps the first minimum.  codes out: int64 [B][n_q][T] with N == B*T; frame n = b*T + t, or
 * n = t*B + b when time_major != 0 (the streaming plans' [T, B, C] layout).
 * work: scratch of rstnet_rvq_encode_workspace(N, ...) bytes; its contents on entry do not matter.
 * Requires dim % 16 == 0, bins % 128 == 0, ldx % 4 == 0, N % T == 0, 0 <= n_q_semantic <= n_q; x, E, Et,
 * enorm and work 16-byte aligned, codes 8-byte aligned (error return otherwise, nothing launched). */
int64_t rstnet_rvq_encode_workspace(int64_t N, int32_t n_q, int32_t dim, int32_t bins);
int rstnet_rvq_encode_f32(const float* x, int64_t ldx, const float* E, const float* Et,
                          const float* enorm, int64_t* codes, void* work, int64_t N, int32_t T,
                          int32_t n_q, int32_t n_q_semantic, int32_t dim, int32_t bins,
                          int32_t time_major, rstnet_stream_t stream);
/* ---- SplitResidualVectorQuantizer.decode gather part (vq.py:317-323; core_vq.py:198-206,
 * 378-384): q [N, 2*dim] = [ E0[c0] | sum_{l>=n_q_semantic} E_l[c_l] ]; the two output_proj are
 * then one rstnet_gemm_rows_f32 with K = 2*dim.  Requires dim % 4 == 0; E and q 16-byte aligned,
 * codes 8-byte aligned (error return otherwise, nothing launched). */
int rstnet_rvq_decode_gather_f32(const int64_t* codes, const float* E, float* q, int64_t N, int32_t T,
                                 int32_t n_q, int32_t n_q_semantic, int32_t dim, int32_t bins,
                                 int32_t time_major, rstnet_stream_t stream);

/* ---- polyphase sinc resampling, fp32: torchaudio.transforms.Resample(orig, new) with its defaults (sinc_interp_hann,
 * lowpass_filter_width 6, rolloff 0.99), which the reference calls wherever it reads audio
 * (MLLM_v2/tools/tokenizer/MimiCodec/mimi_tokenizer.py:40,67; MLLM_v2/egs/moshi_ft/data_scripts/offline_tokenization.py:51;
 * AudioCodec/MimiCodec/inference.py:24-34).  With g = gcd(orig, new), o = orig/g input samples per block, n = new/g
 * output phases per block:
 *   out[r*out_row_stride + q] (q = j*n + p < out_len) = sum_{i<S} xv(r, j*o + x_shift + start[p] + i) * taps[p*S + i]
 *   xv(r, t) = x[r*x_row_stride + t] if 0 <= t < x_len, else 0
 * taps (device fp32 [n][S]) is the fp32 table trimmed to each phase's run of nonzero taps, zero-padded at the end;
 * start (device int32 [n]) the run's first tap, every start[p] in [0, start_max] (a phase outside it is written as NaN).
 * The sum starts at +0.0f and accumulates with fmaf in increasing i, whatever the tiling.
 *   batch form:     x_shift = -w, x_len = L, out_len = ceil(n*L/o) (torchaudio's zero padding is the bounds check);
 *   streaming form: x = a carry buffer, x_shift = 0, x_len = carry + chunk (the two forms are bit-identical).
 * The trimmed table is capped at RSTNET_RESAMPLE_MAX_TABLE_BYTES (n*S*4).  Non-finite input: a NaN / Inf poisons only
 * the outputs whose nonzero run covers it, where torchaudio's full-width conv1d also multiplies it by the zero taps
 * around the run (and so poisons every output whose full window covers it); for finite input the two sums agree up to
 * rounding, and up to the sign of zero. */
#define RSTNET_RESAMPLE_MAX_TABLE_BYTES (48 * 1024)
int rstnet_resample_f32(const float* x, int64_t x_row_stride, int64_t x_len, int64_t x_shift, const float* taps,
                        const int32_t* start, int32_t n, int32_t o, int32_t S, int32_t start_max, float* out,
                        int64_t out_row_stride, int64_t out_len, int32_t rows, rstnet_stream_t stream);

/* ---- codec evaluation over ragged batches of clips.  Clip c of a pack is ref[offsets[c] .. + lengths[c]) and
 * deg[offsets[c] .. + lengths[c]) (device fp32 buffers, device int64 offsets / lengths; the length is already
 * min(len_ref, len_deg)).  Each clip is tiled on its own, from its own frame or sample 0, into fp64 partials in `ws`, and
 * a second launch sums each clip's partials in an order fixed by its length: a clip's sums are the same bytes whatever
 * else is in the pack, where it sits and what the pack's capacity is.  No atomics.  A clip whose length lies outside the
 * host's [min_len, max_len] gets NaN sums; so does a clip with a non-finite sample, and no other clip.
 *
 * The loss sums of one resolution of STFTLoss (Evaluation/codec/compute_ms_stft_loss.py:17-73): torch.stft(x, n_fft, hop,
 * win, hann_window(win)) with center=True, reflect padding (t < 0 -> -t, t >= L -> 2(L-1) - t), the window zero-padded
 * centred to n_fft, onesided; T = sqrt(max(|STFT ref|^2, 1e-7)) ("true"), P the same of deg ("fake").  Frames
 * f = 0 .. L / hop, bins k = 0 .. n_fft / 2.  For each clip c:
 *   sums[(c * n_res + res) * 3 + 0] = sum (T - P)^2      (SpectralConvergence numerator squared, :31)
 *   sums[(c * n_res + res) * 3 + 1] = sum T^2            (its denominator squared, :32)
 *   sums[(c * n_res + res) * 3 + 2] = sum |log P - log T| (LogSTFTMagnitude, :43-45, before the mean), as 0.5 log of the
 *                                                          clamped squares
 * One n_fft-point complex FFT of z = w r + i w d per frame gives both spectra; a frame whose two inputs are equal takes T
 * for P (so a signal against itself gives sums 0 and 2 of exactly 0).  twiddle: device fp32 [n_fft / 2][2],
 * (cos, -sin)(2 pi k / n_fft); window: device fp32 [win], torch.hann_window(win) (periodic); both computed in fp64 and
 * rounded once.  Limits: n_fft a power of two in [64, 4096], 1 <= win <= n_fft, hop >= 1, min_len > n_fft / 2 (torch.stft's
 * reflect padding), clips <= 65535.  ws: rstnet_stft_loss_workspace(clips, max_len, hop) bytes.  Two launches. */
#define RSTNET_STFT_FRAMES_PER_BLOCK 16
int64_t rstnet_stft_loss_workspace(int32_t clips, int64_t max_len, int32_t hop);
int rstnet_stft_loss_sums_f32(const float* ref, const float* deg, const int64_t* offsets, const int64_t* lengths,
                              int32_t clips, int64_t min_len, int64_t max_len, int32_t n_fft, int32_t hop, int32_t win,
                              const float* twiddle, const float* window, double* sums, int32_t n_res, int32_t res,
                              void* ws, int64_t ws_bytes, rstnet_stream_t stream);

/* The moments of SI-SNR (the metric that Evaluation/codec/compute_sisnr.py:11,21 imports as estimate_si_sdr from a
 * module the reference does not ship), per clip in fp64: moments[c * 5 + k] = sum r, sum d, sum r^2, sum d^2, sum r d for
 * k = 0..4 (zeros for an empty clip).  ws: rstnet_sisnr_moments_workspace(clips, max_len) bytes.  Two launches. */
#define RSTNET_SISNR_SAMPLES_PER_BLOCK 8192
int64_t rstnet_sisnr_moments_workspace(int32_t clips, int64_t max_len);
int rstnet_sisnr_moments_f32(const float* ref, const float* deg, const int64_t* offsets, const int64_t* lengths,
                             int32_t clips, int64_t max_len, double* moments, void* ws, int64_t ws_bytes,
                             rstnet_stream_t stream);

/* ======================================================================================
 * Speech-text LM decode step (MLLM_v2/models/llama_streaming.py GPT under `with gpt.streaming(B)`),
 * bf16 activations / weights, fp32 accumulation.  One token per stream: rows are streams.
 * ====================================================================================== */

/* ---- weight-streaming GEMM  out[m,n] = sum_k X[m,k] * W[n,k] (+ R[m,n]), all bf16, W exactly as
 * nn.Linear stores it.  wgmma with W as the 128-row MMA operand (two m64 halves), TMA-staged, fp32
 * accumulator in registers, optional split-K (fp32 partials in `partial_ws` + finalize).  Replaces F.linear
 * in LoRAQKVLinear/LoRALinear after merge (llama_streaming.py:113-143, 368-406), LLaMAMLP
 * (lit_model.py:399-403), lm_head (:691), codecformer_in / multi_linear / gating / audio_linears
 * (llama_streaming.py:727-749, modules/transformer.py:155-179, modules/gating.py:12-21).
 * 1 <= M <= 256, K % 64 == 0 (M > 256 is rejected); each weight tile is read once for all M rows (wgmma N = M
 * rounded up to 16, 32, 64, 128 or 256).  The plan embeds the pointers. */
typedef struct rstnet_skinny_plan rstnet_skinny_plan;
int64_t rstnet_skinny_gemm_workspace(int32_t M, int32_t N, int32_t max_splits);
int rstnet_skinny_gemm_create(const void* X, const void* W, const void* R, void* out, float* partial_ws,
                              int32_t M, int32_t N, int32_t K, int32_t max_splits, rstnet_skinny_plan** plan);
/* Same GEMM with a fused finalize: fin_mode 1: out = bf16(acc + R) AND aux_out = RMSNorm(out) * norm_w (the pre-norm of
 * the following GEMM: Block.forward's `x = attn + x; norm_2(x)`, llama_streaming.py:834-853; kyutai != 0 selects
 * modules/transformer.py:34-48); fin_mode 2: aux_out[m][c] = silu(acc[m][c]) * acc[m][N/2 + c] (LLaMAMLP / ActivationGating),
 * `out` unused.  Both need partial_ws.  fin_mode 3: the same gating for a weight whose rows are INTERLEAVED (row 2c = the
 * gate row c, row 2c + 1 = the value row c): aux_out[m][c] = silu(acc[m][2c]) * acc[m][2c + 1] computed in the GEMM's own
 * epilogue (one K slice, no workspace, no finalize launch); N even. */
int rstnet_skinny_gemm_create_fused(const void* X, const void* W, const void* R, void* out, float* partial_ws,
                                    int32_t M, int32_t N, int32_t K, int32_t max_splits, int32_t fin_mode,
                                    const void* norm_w, void* aux_out, float eps, int32_t kyutai,
                                    rstnet_skinny_plan** plan);
int rstnet_skinny_gemm_run(const rstnet_skinny_plan* plan, rstnet_stream_t stream);
void rstnet_skinny_gemm_destroy(rstnet_skinny_plan* plan);

/* ---- x[b] = sum_cb input_emb[cb][seq[b,cb+1]] + wte[seq[b,0]] with bf16 rounding after every add and
 * an exact zero row for id -1 (GPT.forward_global, llama_streaming.py:680-687; ScaledEmbedding :493-517).
 * seq: int64, row b at seq + b*seq_stride; tables_dev: device array of n_q table pointers. */
/* wte has wte_rows rows, every audio table table_rows rows; an id outside [-1, rows) -> NaN row + error bit 0. */
int rstnet_lm_embed_sum_bf16(const int64_t* seq, int32_t seq_stride, const void* wte, int64_t wte_rows,
                             const void* const* tables_dev, int64_t table_rows, int32_t n_q, int32_t E, void* x, int32_t rows,
                             rstnet_stream_t stream);
/* out[r] = table[ids[r*id_stride]] (zero row for id -1): codecformer_text_emb / codecformer_emb (:738-742) */
int rstnet_lm_embed_rows_bf16(const int64_t* ids, int32_t id_stride, const void* table, int64_t table_rows, int32_t D,
                              void* out, int32_t rows, rstnet_stream_t stream);
/* ---- RMSNorm, fp32 inside.  kyutai == 0: lit_model.RMSNorm (lit_model.py:707-714);
 * kyutai != 0: modules/transformer.py:34-48 `_rms_norm` with dtype=float (eps added before the mean's rsqrt). */
int rstnet_lm_rms_norm_bf16(const void* x, const void* w, void* y, int32_t rows, int32_t dim, float eps, int32_t kyutai,
                            rstnet_stream_t stream);
/* ---- rotate-half RoPE with the model's bf16 cos/sin tables [rope_rows][rope_n] (rope_n = rotary_percentage * hs
 * leading dims rotate, llama_streaming.py:979-982) + ring-KV append (lit_model.py:560-573, 620-634).
 * `rows` = Tn * B (time, stream) pairs, time-major: row r = tl*B + b is stream b at position *offset + tl (a decode step
 * has Tn == 1; a prefill chunk several consecutive positions per stream).  qkv [rows][n_kv][n_head/n_kv + 2][hs] (litgpt
 * per-group interleave, llama_streaming.py:952-963; n_kv == n_head is MHA); q_out [rows][n_head*hs];
 * kv [2][B][n_kv][cap][hs] -- K/V are stored once per KV GROUP (the reference expands them to n_head copies before its
 * cache, :965-967; the attention result is the same).  A position >= rope_rows -> NaN q/k + error bit 1.
 * Row map (ragged prefill of some streams of a live scope, GPT.prefill_streams; serves the prompt pass of
 * infer_no_streaming.py:232-240 for a batch of utterances with different prompt lengths): with row_stream / row_tl given
 * (both or neither; offset_stride must be 1), row r is stream row_stream[r] at position offset[row_stream[r]] + row_tl[r]
 * instead, in any order of (stream, position) pairs, and rows need not be a multiple of B; row_stream[r] == -1 marks a
 * padding row that reads and writes nothing.  Both forms run one compiled kernel.  This is the unpaged case of
 * rstnet_lm_rope_kv_append_paged_bf16 (a contiguous ring per stream); both run the same kernel. */
int rstnet_lm_rope_kv_append_bf16(const void* qkv, const void* cos_tab, const void* sin_tab, int64_t rope_rows, int32_t rope_n,
                                  const int64_t* offset, int32_t offset_stride /* 0 shared, 1 per stream */,
                                  const int32_t* row_stream, const int32_t* row_tl, void* q_out, void* kv, int32_t rows,
                                  int32_t B, int32_t n_head, int32_t n_kv, int32_t hs, int32_t cap, rstnet_stream_t stream);
/* ---- paged KV: the same logical ring (position p in slot p % cap, same mask), stored in pages of P = 2^log2_page
 * positions.  Slot s of stream b lives in page page_table[b * pages_stride + s / P], row s % P, of the pool
 * kv[n_pages][2][n_kv][P][hs] (one pool per layer; a page index names the same positions in every layer, so one table
 * serves them all).  page_table int32 [B][pages_stride] with pages_stride * P >= cap; an entry of -1 is unmapped and never
 * dereferenced: a row whose own position falls on an unmapped page writes nothing (like a padding row).  Every byte
 * stored and every sum is the contiguous form's; only addresses change.  Errors before any launch: a null table, a
 * log2_page outside [RSTNET_KV_LOG2_PAGE_MIN, RSTNET_KV_LOG2_PAGE_MAX], pages_stride * P < cap. */
#define RSTNET_KV_LOG2_PAGE_MIN 4
#define RSTNET_KV_LOG2_PAGE_MAX 12
int rstnet_lm_rope_kv_append_paged_bf16(const void* qkv, const void* cos_tab, const void* sin_tab, int64_t rope_rows,
                                        int32_t rope_n, const int64_t* offset, int32_t offset_stride, const int32_t* row_stream,
                                        const int32_t* row_tl, void* q_out, void* kv, int32_t rows, int32_t B, int32_t n_head,
                                        int32_t n_kv, int32_t hs, int32_t cap, const int32_t* page_table, int32_t pages_stride,
                                        int32_t log2_page, rstnet_stream_t stream);
/* ---- Kyutai pair-RoPE for the Moshi-style LMModel's temporal transformer (models/model.py:364-389; modules/rope.py:11-68,
 * modules/transformer.py:391-399): qkv [rows][3][H][hd] ((p h d) layout); (even, odd) pairs of q / k rotate by
 * freqs[p] * (offset + tl) (freqs [hd/2] fp32 = exp(-ln(max_period) * 2 p / hd), from the host), fp32 inside, one rounding
 * to bf16; rotated q -> q_out [rows][H*hd],
 * rotated k and v -> kv[2][B][H][cap][hd] at slot pos % cap.  Rows / offsets as rstnet_lm_rope_kv_append_bf16. */
int rstnet_lm_rope_pair_kv_append_bf16(const void* qkv, const int64_t* offset, int32_t offset_stride, void* q_out, void* kv,
                                       int32_t rows, int32_t B, int32_t H, int32_t hd, int32_t cap, const float* freqs,
                                       rstnet_stream_t stream);
/* ---- the Kyutai pair-RoPE append over a paged pool kv[n_pages][2][H][P][hd] (page table, its checks and the unmapped
 * rule as rstnet_lm_rope_kv_append_paged_bf16): a row whose own slot is on an unmapped page writes neither q_out nor K/V.
 * Every stored byte equals the contiguous form's; both run the same kernel. */
int rstnet_lm_rope_pair_kv_append_paged_bf16(const void* qkv, const int64_t* offset, int32_t offset_stride, void* q_out, void* kv,
                                             int32_t rows, int32_t B, int32_t H, int32_t hd, int32_t cap, const float* freqs,
                                             const int32_t* page_table, int32_t pages_stride, int32_t log2_page,
                                             rstnet_stream_t stream);
/* ---- the Kyutai pair-RoPE append with a row map over contiguous rings (ragged chunks that pack many utterances:
 * rstnet_b200.moshi.score_many, LMModel.forward): row r is stream row_stream[r] at position offset[row_stream[r]] + row_tl[r]
 * (offset int64 [B], one counter per stream), and row_stream[r] == -1 marks a padding row that reads and writes nothing,
 * neither q_out nor K/V.  The angle is fp32(offset) + fp32(tl) times freqs, as in the uniform form, and every stored byte
 * equals a uniform launch's for the same (stream, position).  Null pointers (either half of the map included), rows < 1 and
 * bad shapes are error returns before any launch.  Same kernel as rstnet_lm_rope_pair_kv_append_bf16.
 * Reference call site: models/model.py:364-389 (forward_text over a whole sequence, modules/transformer.py:391-399). */
int rstnet_lm_rope_pair_kv_append_rows_bf16(const void* qkv, const int64_t* offset, const int32_t* row_stream, const int32_t* row_tl,
                                            void* q_out, void* kv, int32_t rows, int32_t B, int32_t H, int32_t hd, int32_t cap,
                                            const float* freqs, rstnet_stream_t stream);
/* ---- the Kyutai pair-RoPE append with both a row map and a page table (a ragged prompt prefill of some rows of a live
 * paged scope: LMGen.prefill_streams).  Rows, offsets and padding rows as rstnet_lm_rope_pair_kv_append_rows_bf16; the
 * pool, table, its checks and the unmapped rule as rstnet_lm_rope_pair_kv_append_paged_bf16.  Every stored q and K/V byte
 * equals the contiguous row-map form's for the same (stream, position); only addresses change.  Same kernel.
 * Reference call site: moshi/models/lm.py LMGen.step's forward_text, run over the prompt's positions at once
 * (models/model.py:364-389, modules/transformer.py:391-399). */
int rstnet_lm_rope_pair_kv_append_paged_rows_bf16(const void* qkv, const int64_t* offset, const int32_t* row_stream,
                                                  const int32_t* row_tl, void* q_out, void* kv, int32_t rows, int32_t B, int32_t H,
                                                  int32_t hd, int32_t cap, const float* freqs, const int32_t* page_table,
                                                  int32_t pages_stride, int32_t log2_page, rstnet_stream_t stream);
/* ---- one query position per row over the ring with RingKVCache.complete's position labels and the
 * (pos_k>=0)&(delta>=0)&(delta<context) mask (llama_streaming.py:983-992), fp32 softmax. HBM-bound.  Rows and row map as
 * rstnet_lm_rope_kv_append_bf16 (padding rows write no output); every position of the launch must already be in the ring
 * and no slot a query needs may have been overwritten (callers bound Tn as rstnet_b200/lm.py's prefill_chunk and
 * row_chunk_positions do: up to the wrap, then cap - context + 1).  cap < 2 or
 * context < 1 (an empty window) is an error return before any launch.  This is the unpaged
 * case of rstnet_lm_paged_decode_attention_bf16; both run the same kernel. */
int rstnet_lm_ring_decode_attention_bf16(const void* q, const void* kv, const int64_t* offset, int32_t offset_stride,
                                         const int32_t* row_stream, const int32_t* row_tl, void* out, int32_t rows, int32_t B,
                                         int32_t n_head, int32_t n_kv, int32_t hs, int32_t cap, int32_t context,
                                         rstnet_stream_t stream);
/* ---- ring decode attention over a paged pool (page table as rstnet_lm_rope_kv_append_paged_bf16): the same keys in the
 * same order and the same sums, so the output equals the contiguous form's bit for bit.  A row whose own position is
 * on an unmapped page writes an all-zero output; a key slot on an unmapped page is not read (callers keep every key of a
 * query's window mapped).  Same argument checks as the paged append. */
int rstnet_lm_paged_decode_attention_bf16(const void* q, const void* kv, const int64_t* offset, int32_t offset_stride,
                                          const int32_t* row_stream, const int32_t* row_tl, void* out, int32_t rows, int32_t B,
                                          int32_t n_head, int32_t n_kv, int32_t hs, int32_t cap, int32_t context,
                                          const int32_t* page_table, int32_t pages_stride, int32_t log2_page,
                                          rstnet_stream_t stream);
/* out[m][c] = silu(ab[m][c]) * ab[m][I + c]   (LLaMAMLP / ActivationGating) */
int rstnet_lm_silu_mul_bf16(const void* ab, void* out, int32_t M, int32_t I, rstnet_stream_t stream);
/* ---- depth transformer attention at codebook step `step` (keys 0..step, capacity dep_q <= 8, no RoPE):
 * qkv [B][3][H][hd]; kvd [2][B][H][cap][hd] (modules/transformer.py:375-419 with weights_per_step).
 * ring_quirk != 0: streaming form (forward_codecformer, llama_streaming.py:727-749) -- RingKVCache.complete masks key 0
 * on the last step; 0: non-streaming form (forward_local, :694-725; KVCacheResult.from_kv keeps every key). */
int rstnet_lm_depth_attention_bf16(const void* qkv, void* kvd, void* out, int32_t B, int32_t H, int32_t hd, int32_t cap,
                                   int32_t step, int32_t ring_quirk, rstnet_stream_t stream);
/* ---- sample_token / sample_token_audio[_2048] (utils/sampling.py:85-154): row r of logits [rows][V] draws one id
 * among its candidates, the ids < n_valid (<= 0 or > V: all V), into tokens[r * tok_stride].  Modes:
 *   top_k == 0 -> argmax (first maximum; use_sampling False);
 *   1 <= top_k <= 1024 -> top-k + temperature + exponential-noise multinomial (sample_top_k, :49-60; top_k is clamped to
 *     the candidates: torch.topk would raise, the whole support is the natural reading);
 *   top_k < 0 -> temperature multinomial over all candidates (sample_token with top_k == 0, :97-101);
 *   top_k != 0 and 0 < top_p < 1 -> nucleus (sample_top_p, :66-82; it takes precedence over top_k): with
 *     w_i = exp((l_i - max) / temp) over the candidates, id t is kept iff the mass of the ids before it in the order
 *     (logit desc, index asc) is <= top_p * sum(w); equal logits at the cut are kept lowest index first.  The draw is the
 *     first maximum of the top_k < 0 score over the kept ids, so it equals the top_k < 0 draw whenever that draw is kept.
 *     Masses are summed in fixed point (2^-40): identical calls and graph replays give identical tokens.  top_p >= 1 is
 *     the top_k < 0 multinomial; top_p == 0 leaves the mode to top_k.  Unlike the reference's masked audio samplers (NaN
 *     with top_p > 0) the distribution is renormalised over the candidates.
 *   In every mode -0 and +0 are equal logits, a NaN logit is never drawn and takes no top-k slot, and a row in which no
 *   kept id scores above -inf (every candidate -inf or NaN, say) draws id 0: every token is an id in [0, n_valid).
 * Candidates per row (InferenceImp over a batch of utterances, each with its own candidate sets
 * infer_no_streaming.py:264-283): n_valid_rows given, row r samples ids < n_valid_rows[r * n_valid_stride] (<= 0 or > V:
 * all V) in place of the scalar n_valid, with top_k clamped per row.
 * Settings per row: top_k_rows / temp_rows / top_p_rows (all three or none; int32 / fp32 / fp32) give row r the entry at
 * r * param_stride in place of the scalars, so one [rows, 2] table serves the text head (column 0) and the audio heads
 * (column 1).  The tables are read on the device: the caller validates them (top_k <= 1024, temp > 0 where top_k != 0,
 * top_p finite and >= 0).  The scalars are validated here when no table is given.
 * RNG: counter-based, keyed by (seed, *step_counter, r) (step_counter NULL: step 0), or, with step_rows / key_rows given
 * (both or neither; each utterance its own random stream), by (seed, step_rows[r], key_rows[r]).  With key_rows[r] == r,
 * step_rows[r] == *step_counter, one n_valid and the scalars in every row of the tables, the per-row forms draw exactly
 * the tokens of the scalar form: all forms run one compiled kernel. */
int rstnet_lm_sample_params_bf16(const void* logits, int32_t rows, int32_t V, int32_t n_valid, const int32_t* n_valid_rows,
                                 int32_t n_valid_stride, int32_t top_k, float temp, float top_p, const int32_t* top_k_rows,
                                 const float* temp_rows, const float* top_p_rows, int32_t param_stride, uint32_t seed,
                                 const int64_t* step_counter, const int64_t* step_rows, const uint32_t* key_rows,
                                 int64_t* tokens, int32_t tok_stride, rstnet_stream_t stream);

/* ---- teacher-forced scoring: F.cross_entropy(ignore_index, reduction='none'), argmax and the mask sums of
 * CrossEntropyAndAccuracy (models/model.py:31-65) over bf16 logit rows.  Row i (V logits at logits + i * row_stride;
 * any stride >= V, rows need not be 16-byte aligned) belongs to group g = i % groups (the codebook) and to accumulator
 * slot row_slot[i] (NULL: slot 0, n_slots == 1; a negative slot is a padding row: it is not read and adds nothing).
 * Per row (fp32): nll[i] = logsumexp(x) - x[labels[i]], 0 when labels[i] == ignore_ids[g] (ignore_ids may be NULL),
 * NaN when a logit is NaN; pred[i] = torch.argmax (first maximum; a NaN is the maximum).  A label outside [0, V) that is
 * not the ignore id is where F.cross_entropy raises: that row's nll is NaN and error bit 0 is set
 * (rstnet_device_error_flags).
 * Then, in fp64, acc[(slot * groups + g) * 5 + k] += over the slot's rows of group g:
 *   k = 0: sum weights[i] * nll[i]; 1: #(weights != 0); 2: #(weights == 1); 3: #(pred == label and weights != 0);
 *   4: #(pred == label and weights == 1).
 * The sums run in a fixed order (a second launch, no atomics): identical calls give identical bytes.  Two launches,
 * graph-capturable. */
int rstnet_lm_cross_entropy_bf16(const void* logits, int64_t row_stride, int32_t rows, int32_t V, int32_t groups,
                                 const int64_t* labels, const int64_t* ignore_ids, const float* weights,
                                 const int32_t* row_slot, int32_t n_slots, float* nll, int32_t* pred, double* acc,
                                 rstnet_stream_t stream);

/* ---- the acoustic-delay token cache of LMGen.step (models/model.py:490-562; moshi/models/lm.py LMGen.step), per stream:
 * the eager cache writes, input copy, write-back and gather of that step, as two launches around the LM frame.
 * cache [B][K][CT] int64 (K = n_q + 1 codebooks, CT = max_delay + 2); off [B] int64, the stream's step count; active [B]
 * int64 (NULL = every stream active), a stream with 0 is HELD: nothing of its cache, off, valid or out is written;
 * delays [K] int64 (device).  Column indices are taken modulo CT.  Token ids (incl. -1 zero / -2 ungenerated) are copied
 * unchanged.
 * cache_in, before the temporal step: for active streams, user[b][k - dep_q - 1] -> column off + delays[k] of every
 * k > dep_q, then the initial token (text_init for k = 0, audio_init otherwise) -> column off of every k with
 * off <= delays[k]; then seq[b][0..K) = column off for every stream (held streams: ids < -1 become -1).  */
int rstnet_lm_delay_cache_in(int64_t* cache, const int64_t* off, const int64_t* active, const int64_t* delays,
                             const int64_t* user, int32_t user_stride, int64_t* seq, int32_t seq_stride, int32_t B, int32_t K,
                             int32_t dep_q, int32_t CT, int64_t text_init, int64_t audio_init, rstnet_stream_t stream);
/* cache_out, after the last depth sample, active streams: tokens[b][0..dep_q] -> column off + 1; off += 1;
 * out[b][k] = column off - max_delay + delays[k] of k = 0..dep_q; valid[b] = off > max_delay.  CT == max_delay + 2. */
int rstnet_lm_delay_cache_out(int64_t* cache, int64_t* off, const int64_t* active, const int64_t* delays,
                              const int64_t* tokens, int32_t tok_stride, int64_t* out, int32_t out_stride, int64_t* valid,
                              int32_t B, int32_t K, int32_t dep_q, int32_t CT, int32_t max_delay, rstnet_stream_t stream);

/* prompt (LMGen.prefill_streams), n listed rows: row rows[i] runs lengths[i] steps of cache_in then cache_out from its
 * current cache and off, active, with user[k - dep_q - 1] = prompt[(starts[i] + t) * prompt_stride + k] for k > dep_q and
 * tokens[k] = the same entry for k <= dep_q at step t (the prompt in LMGen's step layout, [sum P][K] packed); the seq row
 * cache_in forms at step t -> feed[(starts[i] + t) * feed_stride + k] (the temporal transformer's prefill input).  Then
 * the row's cache columns, off += lengths[i] and valid = off > max_delay are written; `out` is not.  Every byte equals
 * lengths[i] launch pairs of cache_in / cache_out on the row.  A row of length 0 is left untouched.  rows, starts and
 * lengths are int32 HOST arrays, read at the call and carried in the launch's parameters (graph-capturable: a captured
 * launch keeps the list).  Error returns before any launch: a null pointer, n outside [0, RSTNET_DELAY_PROMPT_MAX_ROWS],
 * a bad shape (as cache_out; K * CT * 8 <= 48 KiB) or stride, a row outside [0, B), a row listed twice, a negative start
 * or length.  One CTA per row of nonzero length; nothing is launched when there is none.
 * Reference call site: moshi/models/lm.py LMGen.step (MLLM_v2/moshi/models/lm.py:398-455), P times with the sampled
 * tokens replaced by the prompt's. */
#define RSTNET_DELAY_PROMPT_MAX_ROWS 256
int rstnet_lm_delay_cache_prompt(int64_t* cache, int64_t* off, int64_t* valid, const int64_t* delays, const int64_t* prompt,
                                 int32_t prompt_stride, int64_t* feed, int32_t feed_stride, const int32_t* rows,
                                 const int32_t* starts, const int32_t* lengths, int32_t n, int32_t B, int32_t K, int32_t dep_q,
                                 int32_t CT, int32_t max_delay, int64_t text_init, int64_t audio_init, rstnet_stream_t stream);

/* ---- segment gather / scatter: one batch row's streaming state <-> a packed staging blob (session suspend / resume).
 * A segment is `count` pieces of `bytes` at base + i * stride_bytes (device memory); in staging it occupies
 * [staging_offset, + count * bytes), the pieces back to back.  gather copies every segment into staging, scatter back.
 * `staging` is pinned host memory (reached through UVA; device memory works too); `table` holds n entries in device
 * memory or in pinned host memory, which the kernel reads directly (a device table is copied back to the host for the
 * checks, which synchronises).  One launch of at most `ctas` CTAs.  Accesses are 16 bytes wide where base, stride, piece
 * size and staging address are 16-byte aligned, else 8, 4 or 1.  Checked before any launch, each an error return: n < 0,
 * ctas < 1, a null table / staging / base, count, bytes or staging_offset < 0, two segments whose staging ranges
 * overlap, and (scatter) a segment whose pieces overlap in device memory.  n == 0 launches nothing. */
typedef struct {
  void* base;
  int64_t stride_bytes;
  int64_t bytes;
  int32_t count;
  int64_t staging_offset;
} rstnet_segment;
int rstnet_segments_gather(const rstnet_segment* table_dev, int32_t n, void* staging, int32_t ctas, rstnet_stream_t s);
int rstnet_segments_scatter(const rstnet_segment* table_dev, int32_t n, const void* staging, int32_t ctas, rstnet_stream_t s);

/* ---- batched KV page copy (paged decode scopes; added in version 206): for every pool i < n_pools (pools[i], one per
 * layer, a host array of device pointers) and every pair j < n_pairs, the page_bytes at pools[i] + pairs[2j] * page_bytes
 * are copied to pools[i] + pairs[2j + 1] * page_bytes.  `pairs` (int32 (src, dst) pairs) is device memory or pinned host
 * memory, which the kernel reads directly; a device table is copied back to the host for the checks, which synchronises,
 * so a launch that a stream captures into a graph takes a pinned host table (its entries are read at every replay).  One
 * launch of at most `ctas` CTAs; accesses are 16 bytes wide where the pool base and page_bytes are 16-byte aligned, else 8,
 * 4 or 1.  Checked before any launch, each an error return: a null pools / pairs / pool pointer, n_pools outside
 * [1, RSTNET_KV_COPY_MAX_POOLS], n_pairs < 0, page_bytes <= 0, ctas < 1, a negative page index, src == dst, a page that
 * is the dst of two pairs or both a src and a dst.  Page indices are not checked against the pool size (the caller's, as
 * with the page table).  n_pairs == 0 launches nothing. */
#define RSTNET_KV_COPY_MAX_POOLS 256
int rstnet_kv_pages_copy(const void* const* pools, int32_t n_pools, const int32_t* pairs, int32_t n_pairs, int64_t page_bytes,
                         int32_t ctas, rstnet_stream_t s);

/* ---- generation window of the batch generation loop, advanced after the last depth sample of a frame (graph-capturable;
 * MLLM_v2/infer_no_streaming.py:264-292).  rec [B][RSTNET_GEN_REC] int32 (device): {pre_gen_len, minlen, maxlen, g_idx,
 * mode}; g_idx is the frame these tokens are; mode & 3 is RSTNET_GEN_HELD / _FIXED / _WINDOWED, | RSTNET_GEN_ARGMAX for a
 * row that takes the whole card.  tokens [B][tok_stride] int64 (text, then audio codebooks 0 .. dep_q - 1).  Per row:
 *   held:                                               status = IDLE; nothing else is written;
 *   windowed, g_idx > minlen and a token >= 2048 in audio codebooks 3 .. 7: status = STOPPED (the frame is dropped), the
 *                                                       row becomes held;
 *   otherwise g_idx + 1 >= maxlen:                      status = LAST (the frame is kept), the row becomes held;
 *   otherwise:                                          status = RUNNING, g_idx += 1, and row_valid[b][0 .. dep_q) gets
 *     the next frame's candidate counts: `card` for an argmax row, else 2049 for l > 0 when pre_gen_len + g_idx > minlen,
 *     2048 otherwise.
 * status [B] int32 (device).  Checked before any launch, each an error return: a null pointer, B < 1, dep_q < 1,
 * card < 2049, tok_stride < dep_q + 1, valid_stride < dep_q. */
#define RSTNET_GEN_REC 5
enum { RSTNET_GEN_HELD = 0, RSTNET_GEN_FIXED = 1, RSTNET_GEN_WINDOWED = 2, RSTNET_GEN_ARGMAX = 4 };
enum { RSTNET_GEN_RUNNING = 0, RSTNET_GEN_LAST = 1, RSTNET_GEN_STOPPED = 2, RSTNET_GEN_IDLE = 3 };
int rstnet_lm_gen_rows_advance(const int64_t* tokens, int32_t tok_stride, int32_t* rec, int32_t* row_valid, int32_t valid_stride,
                               int32_t* status, int32_t B, int32_t dep_q, int32_t card, rstnet_stream_t stream);

/* ---- forced tokens (added in version 206): run after the sampler of head `col` (graph-capturable).  For every row
 * r < rows, tokens[r * tok_stride + col] = force[r * force_stride + col] where that id is >= 0; a negative id keeps the
 * sampled token.  An id >= V (the head's vocabulary) is not written and sets the sticky device error bit 1
 * (rstnet_device_error_flags).  tokens int64 and force int32, device memory.  Checked before any launch, each an error
 * return: a null pointer, rows < 1, V < 1, col < 0, col >= tok_stride or col >= force_stride.  One thread per row. */
int rstnet_lm_force_tokens(int64_t* tokens, int32_t tok_stride, int32_t col, const int32_t* force, int32_t force_stride,
                           int32_t rows, int32_t V, rstnet_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* RSTNET_B200_H */
