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
 * The kernel is persistent (at most one CTA per SM walking the 128 x 32 or 128 x 64 output tiles).  ELU, as pre- and
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
/* the plan's tile grid: M tiles (I tiles x O_out), N tiles, tile width */
int rstnet_tc_gemm_grid(const rstnet_tc_plan* plan, int32_t* grid_x, int32_t* grid_y, int32_t* tile_n);
/* hi[i] = tf32_rna(x[i]); lo[i] = tf32_rna(x[i] - hi[i])  (one-time weight preparation for precision 0) */
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
 * work: scratch of rstnet_rvq_encode_workspace(N, ...) bytes. */
int64_t rstnet_rvq_encode_workspace(int64_t N, int32_t n_q, int32_t dim, int32_t bins);
int rstnet_rvq_encode_f32(const float* x, int64_t ldx, const float* E, const float* Et,
                          const float* enorm, int64_t* codes, void* work, int64_t N, int32_t T,
                          int32_t n_q, int32_t n_q_semantic, int32_t dim, int32_t bins,
                          int32_t time_major, rstnet_stream_t stream);
/* ---- SplitResidualVectorQuantizer.decode gather part (vq.py:317-323; core_vq.py:198-206,
 * 378-384): q [N, 2*dim] = [ E0[c0] | sum_{l>=n_q_semantic} E_l[c_l] ]; the two output_proj are
 * then one rstnet_gemm_rows_f32 with K = 2*dim. */
int rstnet_rvq_decode_gather_f32(const int64_t* codes, const float* E, float* q, int64_t N, int32_t T,
                                 int32_t n_q, int32_t n_q_semantic, int32_t dim, int32_t bins,
                                 int32_t time_major, rstnet_stream_t stream);

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
 * 1 <= M <= 128, K % 64 == 0.  The plan embeds the pointers. */
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
 * cache, :965-967; the attention result is the same).  A position >= rope_rows -> NaN q/k + error bit 1. */
int rstnet_lm_rope_kv_append_bf16(const void* qkv, const void* cos_tab, const void* sin_tab, int64_t rope_rows, int32_t rope_n,
                                  const int64_t* offset, int32_t offset_stride /* 0 shared, 1 per stream */, void* q_out,
                                  void* kv, int32_t rows, int32_t B, int32_t n_head, int32_t n_kv, int32_t hs, int32_t cap,
                                  rstnet_stream_t stream);
/* ---- Kyutai pair-RoPE for the Moshi-style LMModel's temporal transformer (models/model.py:364-389; modules/rope.py:11-68,
 * modules/transformer.py:391-399): qkv [rows][3][H][hd] ((p h d) layout); (even, odd) pairs of q / k rotate by
 * freqs[p] * (offset + tl) (freqs [hd/2] fp32 = exp(-ln(max_period) * 2 p / hd), from the host), fp32 inside, one rounding
 * to bf16; rotated q -> q_out [rows][H*hd],
 * rotated k and v -> kv[2][B][H][cap][hd] at slot pos % cap.  Rows / offsets as rstnet_lm_rope_kv_append_bf16. */
int rstnet_lm_rope_pair_kv_append_bf16(const void* qkv, const int64_t* offset, int32_t offset_stride, void* q_out, void* kv,
                                       int32_t rows, int32_t B, int32_t H, int32_t hd, int32_t cap, const float* freqs,
                                       rstnet_stream_t stream);
/* ---- one query position per row over the ring with RingKVCache.complete's position labels and the
 * (pos_k>=0)&(delta>=0)&(delta<context) mask (llama_streaming.py:983-992), fp32 softmax. HBM-bound.  Rows as above;
 * every position of the launch must already be in the ring and no slot a query needs may have been overwritten
 * (callers keep *offset + Tn <= cap for Tn > 1).
 * split_ws (optional, rstnet_lm_attention_split_workspace bytes, its first rows*n_head int32 zeroed ONCE by the caller): lets
 * the kernel cut every job's keys in three chunks walked by persistent CTAs when rows * heads would otherwise leave a badly
 * filled last wave; partials are combined in chunk order (deterministic). */
int64_t rstnet_lm_attention_split_workspace(int32_t rows, int32_t n_head, int32_t hs);
int rstnet_lm_ring_decode_attention_bf16(const void* q, const void* kv, const int64_t* offset, int32_t offset_stride,
                                         void* out, int32_t rows, int32_t B, int32_t n_head, int32_t n_kv, int32_t hs,
                                         int32_t cap, int32_t context, void* split_ws, rstnet_stream_t stream);
/* out[m][c] = silu(ab[m][c]) * ab[m][I + c]   (LLaMAMLP / ActivationGating) */
int rstnet_lm_silu_mul_bf16(const void* ab, void* out, int32_t M, int32_t I, rstnet_stream_t stream);
/* ---- depth transformer attention at codebook step `step` (keys 0..step, capacity dep_q <= 8, no RoPE):
 * qkv [B][3][H][hd]; kvd [2][B][H][cap][hd] (modules/transformer.py:375-419 with weights_per_step).
 * ring_quirk != 0: streaming form (forward_codecformer, llama_streaming.py:727-749) -- RingKVCache.complete masks key 0
 * on the last step; 0: non-streaming form (forward_local, :694-725; KVCacheResult.from_kv keeps every key). */
int rstnet_lm_depth_attention_bf16(const void* qkv, void* kvd, void* out, int32_t B, int32_t H, int32_t hd, int32_t cap,
                                   int32_t step, int32_t ring_quirk, rstnet_stream_t stream);
/* ---- the depth transformer of a frame as ONE persistent (cooperative) kernel: steps [k_begin, k_end) of
 * GPT.forward_codecformer (llama_streaming.py:727-749; per-step weights modules/transformer.py:155-179, 518-577; gating
 * modules/gating.py:12-21), each = codecformer_in[k](transformer_out) + embedding of the step's input token, L layers
 * (RMSNorm-f32, per-step in/out projections, attention over the <= dep_q keys of this frame, SiLU gating), audio_linears[k]
 * -> logits[k][M][card], and (do_sample) sample_token_audio on the device: tokens[m][k + 1] feeds step k + 1.
 * tokens[m][k] is the INPUT token of step k (column 0: the text token).  All buffers are the caller's; `barrier` is two
 * uint32 words (arrival counter, zeroed by run; sticky error word: bit 0 token id outside its table, bit 2 barrier
 * watchdog).  w_gin[l*Q + k]: gating linear_in with its rows interleaved in 8-row groups [a_8u..8u+7; b_8u..8u+7] and the
 * hidden width zero-padded to Hp (a multiple of 128); w_gout[l*Q + k]: linear_out [D][Hp].  Requires M <= 128,
 * D, E, Hp multiples of 128, D <= 2048.  step0_embedding (optional, [M][D]) replaces the token lookup of step 0
 * (forward_local passes features there, llama_streaming.py:700-705); ring_quirk as in rstnet_lm_depth_attention_bf16. */
typedef struct rstnet_depth_plan rstnet_depth_plan;
typedef struct {
  int32_t M, D, E, Hp, H, hd, Q, L, card, tok_stride;
  const void* tout; void* x; void* qkv; void* att; void* dh; void* logits; void* dkv; float* ss_part; int64_t* tokens; void* barrier;
  const void* w_in[8]; const void* emb[8]; int64_t emb_rows[8]; const void* w_head[8];
  const void* w_qkv[8]; const void* w_out[8]; const void* a1[8]; const void* a2[8];
  const void* w_gin[64]; const void* w_gout[64];
} rstnet_depth_frame_desc;
int rstnet_lm_depth_frame_create(const rstnet_depth_frame_desc* desc, rstnet_depth_plan** plan);
int rstnet_lm_depth_frame_run(const rstnet_depth_plan* plan, int32_t k_begin, int32_t k_end, int32_t ring_quirk, int32_t do_sample,
                              int32_t top_k, float temp, uint32_t seed, const int64_t* frame_counter, const int32_t* n_valid,
                              const void* step0_embedding, rstnet_stream_t stream);
void rstnet_lm_depth_frame_destroy(rstnet_depth_plan* plan);
/* profiling aid: CTA 0 writes clock64 stamps (start, then after every phase and after every barrier) to trace[>= 1024] */
void rstnet_lm_depth_frame_set_trace(rstnet_depth_plan* plan, int64_t* trace);

/* ---- sample_token / sample_token_audio[_2048] (utils/sampling.py:85-154): ids restricted to [0, n_valid);
 * top_k == 0 -> argmax (first maximum; use_sampling False); 1 <= top_k <= 1024 -> top-k + temperature +
 * exponential-noise multinomial (sample_top_k, :49-60); top_k < 0 -> temperature multinomial over all n_valid ids
 * (sample_token with top_k == 0, :97-101).  Counter-based RNG keyed by (seed, *step_counter, row).
 * tokens[row*tok_stride] = id. */
int rstnet_lm_sample_bf16(const void* logits, int32_t rows, int32_t V, int32_t n_valid, int32_t top_k, float temp,
                          uint32_t seed, const int64_t* step_counter, int64_t* tokens, int32_t tok_stride,
                          rstnet_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* RSTNET_B200_H */
