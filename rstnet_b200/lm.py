"""H100-native decode path of the speech-text LM behind the reference's Python API.

Mirrors ``models.llama_streaming.GPT`` (MLLM_v2/models/llama_streaming.py:520-766):
  * streaming (`with gpt.streaming(B):`): ``forward_global(seq[B,9,T]) -> (transformer_out[B,T,E], text_logits[B,T,V])``
    (:665-692) -- T == 1 is the decode step, T > 1 a prefill chunk (T consecutive positions per stream, the KV ring
    written in one pass; equal to T single-step calls);
  * ``with gpt.codecformer.streaming(B): forward_codecformer(k, prev[B,1,1], transformer_out)`` (:727-749);
  * outside a streaming scope ``forward_global`` is the reference's non-streaming form (positions 0..T-1, nothing kept) and
    ``forward_local(local_start_token, sequence, transformer_out) -> logits[B,T,8,card]`` (:694-725) the teacher-forced
    depth transformer -- the two calls `infer_no_streaming.py:232-308` makes;
  * ``_get_initial_token``, ``codecformer_text_emb``, token-id properties, identical state_dict keys (LoRA keys
    ``...lora_A / lora_B`` are merged into the base weights on load, :113-143, 368-406, 1120-1124);
  * MHA and GQA (``n_query_groups``), partial rotary (``rotary_percentage``), Llama-3.1 ``rope_adjustments``;
plus ``forward_step`` -- the whole frame (temporal step, text sampling, 8 depth steps with sampling) as one CUDA-graph
replay; BASELINE.json names it although no such symbol exists upstream.

All arithmetic runs in librstnet_b200.so: wgmma weight-streaming GEMMs, ring decode attention, fused
norm / RoPE / gating / sampling kernels.  bf16 weights and activations, fp32 accumulation, exactly the
dtype recipe of `GPT(config).to(device, bfloat16)` (infer_no_streaming.py:104-105).
"""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import torch
from torch import nn

from . import _lib, ops
from ._lib import RstnetError
from .codec import _register, on_own_device

MAX_ROWS = 128   # rows (stream, position) pairs per launch of a prefill chunk or a forward_local slice
MAX_STREAMS = 256   # streams of one decode scope (one position each): the widest weight-streaming GEMM reads each weight
                    # tile once for up to 256 rows
ROW_BUCKETS = (16, 32, 64, 128)   # launch widths of a ragged prefill chunk (padding rows fill the rest): one chunk state and
                                  # one set of GEMM plans per width


@dataclass
class Config:
    """The fields of models.llama_streaming.Config the decode path reads (same names / defaults)."""
    block_size: int = 4096
    n_layer: int = 16
    n_embd: int = 4096
    n_head: int = 32
    n_query_groups: Optional[int] = None
    head_size: Optional[int] = None
    intermediate_size: int = 11008
    norm_eps: float = 1e-5
    rope_base: int = 10000
    rotary_percentage: float = 1.0
    rope_condense_ratio: int = 1
    rope_adjustments: Optional[dict] = None
    padded_vocab_size: int = 152064
    audio_card: int = 2048
    n_q: int = 9
    dep_q: int = 8
    codecformer_dim: int = 1024
    codecformer_heads: int = 32
    codecformer_layers: int = 6
    codecformer_dim_feedforward: int = 1024
    context: int = 3000
    # LoRA (llama_streaming.py:447-470): only used to merge lora_A / lora_B found in a checkpoint
    lora_r: int = 0
    lora_alpha: int = 1
    lora_dropout: float = 0.0
    lora_query: bool = False
    lora_key: bool = False
    lora_value: bool = False
    lora_projection: bool = False
    lora_mlp: bool = False
    lora_head: bool = False

    def __post_init__(self):
        if self.head_size is None:
            self.head_size = self.n_embd // self.n_head
        if self.n_query_groups is None:
            self.n_query_groups = self.n_head
        if self.n_head % self.n_query_groups != 0:
            raise ValueError("n_head must be a multiple of n_query_groups")

    @property
    def rope_n_elem(self) -> int:   # config.py:113
        return int(self.rotary_percentage * self.head_size)

    @property
    def ff_hidden(self) -> int:  # modules/gating.py:40-43
        d, ff = self.codecformer_dim, self.codecformer_dim_feedforward
        return (21 * d) // 8 if ff == 4 * d else (2 * ff) // 3


def interleave_gate_rows(w_gate: torch.Tensor, w_value: torch.Tensor) -> torch.Tensor:
    """[gate row 0, value row 0, gate row 1, value row 1, ...]: the packing the GEMM's in-epilogue SiLU gating expects (the
    two rows of an output column sit in neighbouring lanes of the GEMM epilogue; fc_1 / fc_2 of LLaMAMLP,
    lit_model.py:399-403, or the halves of ActivationGating.linear_in, modules/gating.py:12-21)."""
    return torch.stack([w_gate, w_value], dim=1).reshape(2 * w_gate.shape[0], w_gate.shape[1]).contiguous()


class SkinnyGemm:
    """rstnet_skinny_gemm_* plan: out[m,n] = sum_k X[m,k] W[n,k] (+ R[m,n]), bf16, optionally with a fused finalize:
    norm_w/aux -> aux = RMSNorm(out) * norm_w (the next GEMM's pre-norm); silu_out -> silu_out = silu(a) * b, with
    [a; b] = the two halves of the result or, `interleaved` (see `interleave_gate_rows`), its even / odd columns -- the latter
    is finished in the GEMM's epilogue without a finalize launch."""

    def __init__(self, X: torch.Tensor, W: torch.Tensor, out: Optional[torch.Tensor], R: Optional[torch.Tensor],
                 ws: Optional[torch.Tensor], max_splits: int = 8, norm_w: Optional[torch.Tensor] = None,
                 aux: Optional[torch.Tensor] = None, eps: float = 0.0, kyutai: bool = False, silu_out: Optional[torch.Tensor] = None,
                 interleaved: bool = False):
        M, K = X.shape
        N = W.shape[0]
        assert W.shape[1] == K and X.dtype == W.dtype == torch.bfloat16 and X.is_contiguous() and W.is_contiguous()
        if N % 4 != 0:
            ws = None  # split-K / fused finalize work on 4-element groups
        mode = (3 if interleaved else 2) if silu_out is not None else (1 if norm_w is not None else 0)
        if mode in (1, 2) and ws is None:
            raise RstnetError("fused finalize needs a workspace and N % 4 == 0")
        aux_t = silu_out if mode >= 2 else aux
        self._keep = (X, W, out, R, ws, norm_w, aux_t)
        self._h = C.c_void_p()
        self.flops = 2.0 * M * N * K
        self.bytes = 2.0 * (N * K + M * K + M * N)
        p = lambda t: None if t is None else t.data_ptr()
        _lib.check(_lib.lib().rstnet_skinny_gemm_create_fused(p(X), p(W), p(R), p(out), p(ws), M, N, K,
                                                              max_splits if ws is not None else 1, mode, p(norm_w), p(aux_t),
                                                              float(eps), int(kyutai), C.byref(self._h)), "skinny_gemm_create")

    def run(self):
        _lib.check(_lib.lib().rstnet_skinny_gemm_run(self._h, ops._stream()), "skinny_gemm_run")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().rstnet_skinny_gemm_destroy(h)
            except Exception:
                pass
            self._h = None


class _DepthScope:
    """Stand-in for `gpt.codecformer` (a StreamingTransformer upstream): `with gpt.codecformer.streaming(B):`
    starts the per-frame depth state (llama_streaming.py:581: the subtree is fenced from the outer scope)."""

    def __init__(self, gpt: "GPT"):
        self._gpt = gpt

    @contextmanager
    def streaming(self, batch_size: int):
        st = self._gpt._state
        if st is None or st.B != batch_size:
            raise RstnetError("enter gpt.streaming(B) with the same batch size first")
        st.depth_step = 0
        try:
            yield
        finally:
            st.depth_step = None


# --------------------------------------------------------------------------------------- LoRA merge (host, once)
def _lora_delta_qkv(A: torch.Tensor, B: torch.Tensor, c: Config, scaling: float, out_features: int) -> torch.Tensor:
    """LoRAQKVLinear.get_lora_AB (llama_streaming.py:368-380 with conv1d :330-366 and zero_pad :255-328): one rank-r
    update per enabled part of (q, k, v); the parts' rows are scattered to the per-group interleaved layout."""
    enable = (c.lora_query, c.lora_key, c.lora_value)
    n_en = sum(enable)
    r = A.shape[0] // n_en
    hs, nh, nkv = c.head_size, c.n_head, c.n_query_groups
    shapes = [s for s, e in zip((hs * nh, hs * nkv, hs * nkv), enable) if e]
    parts = [Bp @ Ap for Ap, Bp in zip(A.split(r, dim=0), B.split(shapes, dim=0))]
    lora = torch.cat(parts, dim=0) * scaling                                        # [sum(shapes), in]
    group = nh // nkv + 2
    rows = torch.arange(out_features)
    slot = (rows // hs) % group
    ind = []
    if enable[0]:
        ind.append(rows[slot < group - 2])
    if enable[1]:
        ind.append(rows[slot == group - 2])
    if enable[2]:
        ind.append(rows[slot == group - 1])
    ind = torch.cat(ind)
    delta = lora.new_zeros(out_features, lora.shape[1])
    delta.index_copy_(0, ind.to(lora.device), lora)
    return delta


def merge_lora_weights(model: "GPT") -> None:
    """llama_streaming.merge_lora_weights (:1120-1124).  LoRA factors are merged when a checkpoint is loaded, so a GPT
    here is always in the merged state; kept for call-site compatibility."""
    return None


class GPT(nn.Module):
    def __init__(self, config: Config, device=None, dtype=None):
        """device/dtype: create the (random-init) parameters directly there (a 7B model in bf16 on the GPU
        without a 28 GB fp32 host copy); default = CPU fp32 like the reference constructor."""
        super().__init__()
        c = self.config = config
        E, V, I, D, H = c.n_embd, c.padded_vocab_size, c.intermediate_size, c.codecformer_dim, c.ff_hidden
        g = torch.Generator(device=device if device is not None else "cpu").manual_seed(0)
        fk = dict(device=device, dtype=dtype)

        def w_(*shape):
            return torch.empty(*shape, **fk).normal_(0.0, 0.02, generator=g)

        def ones(*shape):
            return torch.ones(*shape, **fk)

        _register(self, "lm_head.linear.weight", w_(V, E))
        _register(self, "transformer.wte.weight", w_(V, E))
        for l in range(c.n_layer):
            p = f"transformer.h.{l}"
            _register(self, f"{p}.norm_1.weight", ones(E))
            _register(self, f"{p}.attn.attn.linear.weight", w_((c.n_head + 2 * c.n_query_groups) * c.head_size, E))
            _register(self, f"{p}.attn.proj.linear.weight", w_(E, c.n_head * c.head_size))
            _register(self, f"{p}.norm_2.weight", ones(E))
            _register(self, f"{p}.mlp.fc_1.linear.weight", w_(I, E))
            _register(self, f"{p}.mlp.fc_2.linear.weight", w_(I, E))
            _register(self, f"{p}.mlp.proj.linear.weight", w_(E, I))
        _register(self, "transformer.ln_f.weight", ones(E))
        for i in range(c.n_q):
            _register(self, f"input_emb.{i}.weight", w_(c.audio_card + 1, E))
        for i in range(c.dep_q):
            _register(self, f"codecformer_in.{i}.weight", w_(D, E))
        for i in range(c.dep_q - 1):
            _register(self, f"codecformer_emb.{i}.weight", w_(c.audio_card + 1, D))
        _register(self, "codecformer_text_emb_.weight", w_(V, D))
        for l in range(c.codecformer_layers):
            p = f"codecformer_.layers.{l}"
            _register(self, f"{p}.self_attn.in_proj_weight", w_(c.dep_q * 3 * D, D))
            _register(self, f"{p}.self_attn.out_proj.weight", w_(c.dep_q * D, D))
            _register(self, f"{p}.norm1.alpha", ones(1, 1, D))
            _register(self, f"{p}.norm2.alpha", ones(1, 1, D))
            for k in range(c.dep_q):
                _register(self, f"{p}.gating.{k}.linear_in.weight", w_(2 * H, D))
                _register(self, f"{p}.gating.{k}.linear_out.weight", w_(D, H))
        for i in range(c.dep_q):
            _register(self, f"audio_linears.{i}.weight", w_(c.audio_card, D))
        self.max_seq_length = c.block_size
        self.codecformer = _DepthScope(self)
        self._state: Optional["_LMState"] = None
        self._packed = None
        self._local_states: Dict[int, "_LMState"] = {}
        self._ns_state: Optional["_LMState"] = None      # scratch scope of the non-streaming forward_global
        self.use_cuda_graphs = True

    # parameter names of the depth transformer (the Moshi-style LMModel of rstnet_b200/moshi.py has the same structure under
    # other names, models/model.py:188-224)
    _DN = dict(din="codecformer_in.{}.weight", demb="codecformer_emb.{}.weight", dtext="codecformer_text_emb_.weight",
               dlayer="codecformer_.layers.{}", dhead="audio_linears.{}.weight")

    # ---- state_dict keys identical to the reference (`codecformer.` / `codecformer_text_emb.` subtrees are
    # stored under private attribute names because `codecformer` / `codecformer_text_emb` are API objects here)
    _RENAME = (("codecformer_.", "codecformer."), ("codecformer_text_emb_.", "codecformer_text_emb."))

    def state_dict(self, *a, **kw):
        sd = super().state_dict(*a, **kw)
        out = type(sd)()
        for k, v in sd.items():
            for src, dst in self._RENAME:
                if k.startswith(src):
                    k = dst + k[len(src):]
            out[k] = v
        return out

    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        sd, lora = {}, {}
        old = {"lm_head.weight": "lm_head.linear.weight"}  # llama_streaming.py:762-766 compatibility mapping
        for k, v in state_dict.items():
            k = old.get(k, k)
            for src, dst in self._RENAME:
                if k.startswith(dst):
                    k = src + k[len(dst):]
            for a, b in ((".attn.weight", ".attn.linear.weight"), (".proj.weight", ".proj.linear.weight"),
                         (".fc_1.weight", ".fc_1.linear.weight"), (".fc_2.weight", ".fc_2.linear.weight")):
                if k.endswith(a) and k.startswith("transformer.h."):
                    k = k[: -len(a)] + b  # base-checkpoint names (llama_streaming.py:1000-1009, 1034-1043)
            if k.endswith(".lora_A") or k.endswith(".lora_B"):
                lora[k] = v
            else:
                sd[k] = v
        self._merge_lora(sd, lora)
        self._packed = None
        self._local_states, self._ns_state = {}, None
        return super().load_state_dict(sd, strict=strict, **kw)

    def _merge_lora(self, sd, lora):
        """W += (B @ A) * (lora_alpha / r) for every wrapped linear that carries LoRA factors: LoRALinear.merge /
        LoRAQKVLinear.merge (llama_streaming.py:113-133, 382-385), i.e. what merge_lora_weights (:1120-1124) leaves behind."""
        c = self.config
        for ka in [k for k in lora if k.endswith(".lora_A")]:
            base = ka[: -len(".lora_A")]
            kb, kw_ = base + ".lora_B", base + ".linear.weight"
            if kb not in lora or kw_ not in sd:
                raise RuntimeError(f"LoRA factors for {base} without a matching lora_B / base weight")
            A, B = lora[ka].float(), lora[kb].float()
            W = sd[kw_]
            if base.endswith(".attn.attn"):
                n_en = sum((c.lora_query, c.lora_key, c.lora_value))
                if n_en == 0:
                    raise RuntimeError("the checkpoint holds QKV LoRA factors but Config.lora_query/key/value are all False")
                r = A.shape[0] // n_en
                delta = _lora_delta_qkv(A, B, c, c.lora_alpha / r, W.shape[0])
            else:
                r = A.shape[0]
                delta = (B @ A) * (c.lora_alpha / r)
            sd[kw_] = (W.float() + delta.to(W.device)).to(W.dtype)   # in-place add into the weight's dtype upstream (:133)

    def _apply(self, fn, *a, **kw):
        self._packed = None
        self._local_states, self._ns_state = {}, None
        return super()._apply(fn, *a, **kw)

    # ---- token-id conventions (llama_streaming.py:590-634)
    @property
    def zero_token_id(self) -> int:
        return -1

    @property
    def text_initial_token_id(self) -> int:
        return 151655

    @property
    def initial_token_id(self) -> int:
        return self.config.audio_card

    @property
    def num_codebooks(self) -> int:
        return self.config.n_q + 1

    @property
    def num_audio_codebooks(self) -> int:
        return self.config.n_q

    @property
    def audio_offset(self) -> int:
        return 1

    @property
    def ungenerated_token_id(self) -> int:
        return -2

    @property
    def device(self):
        return next(iter(self.parameters())).device

    def _get_initial_token(self) -> torch.Tensor:
        tok = torch.full([1, self.num_codebooks, 1], self.initial_token_id, device=self.device, dtype=torch.long)
        tok[:, 0] = self.text_initial_token_id
        return tok

    def codecformer_text_emb(self, ids: torch.Tensor) -> torch.Tensor:
        w = dict(self.named_parameters())["codecformer_text_emb_.weight"]
        y = torch.nn.functional.embedding(ids.clamp(min=0), w)
        return torch.where((ids == self.zero_token_id)[..., None], torch.zeros(1, dtype=y.dtype, device=y.device), y)

    # ---- StreamingModule protocol (modules/streaming.py:33-151)
    def _check_runnable(self):
        dev = self.device
        if dev.type != "cuda":
            raise RstnetError("GPT decode runs on CUDA only (sm_90a kernels; the CPU path is the reference itself)")
        if next(self.parameters()).dtype != torch.bfloat16:
            raise RstnetError("GPT decode runs in bfloat16: call .to(device, torch.bfloat16) as infer_no_streaming.py:104-105 does")

    @property
    def is_streaming(self) -> bool:
        return self._state is not None

    @on_own_device
    def streaming_forever(self, batch_size: int):
        self._check_runnable()
        self._state = _LMState(self, batch_size)

    @contextmanager
    def streaming(self, batch_size: int):
        self.streaming_forever(batch_size)
        try:
            yield
        finally:
            self._state = None

    @on_own_device
    def reset_streaming(self, streams=None):
        """reset_streaming (modules/streaming.py:115-126); `streams` (extension) restarts only those batch rows: their
        position counters go back to 0 (the ring contents need no clearing: the position mask hides them)."""
        if self._state is None:
            raise ValueError("Trying to reset streaming, but the model wasn't streaming.")
        self._state.reset(streams)

    def set_active_streams(self, mask) -> None:
        """Extension for batched serving: hold the rows whose flag is 0 during the following steps (see codec.py)."""
        if self._state is None:
            raise ValueError("the model is not streaming")
        self._state.set_active(mask)

    def get_streaming_state(self):
        """modules/streaming.py:128-136: name -> state object; the whole LM is one streaming module here."""
        return {"": self._state}

    def set_streaming_state(self, state):
        """modules/streaming.py:138-151."""
        state = dict(state)
        if "" not in state:
            raise RuntimeError("Expected to find a streaming state for .")
        st = state.pop("")
        if state:
            raise RuntimeError(f"Some states were not consumed: {list(state.keys())}")
        if st is not None and (not isinstance(st, _LMState) or st.m is not self):
            raise RuntimeError("the streaming state belongs to another model")
        self._state = st

    def check_device_errors(self, clear: bool = True) -> None:
        """Raise if a kernel met an input the reference would have raised on (out-of-range token id, position beyond
        block_size): device code cannot raise, it poisons its output and sets a sticky flag (synchronises)."""
        with torch.cuda.device(self.device):
            flags = int(_lib.lib().rstnet_device_error_flags(int(clear)))
        if flags & 1:
            raise IndexError("a token id was outside its embedding table (index out of range in self)")
        if flags & 2:
            raise IndexError(f"a position reached block_size = {self.config.block_size} (RoPE table exhausted)")

    # ---- reference API
    @torch.no_grad()
    @on_own_device
    def forward_global(self, sequence: torch.Tensor):
        B, K, T = sequence.shape
        assert K == self.num_codebooks, f"Sequence shape {sequence.shape} must match the number of codebooks."
        if self.max_seq_length < T:
            raise ValueError(f"Cannot forward sequence of length {T}, max seq length is only {self.max_seq_length}.")
        if self._state is None:
            # non-streaming form (CausalSelfAttention.forward with state None, llama_streaming.py:946-998): positions
            # 0..T-1 from scratch, nothing is kept afterwards
            self._check_runnable()
            if T > self.config.context:
                raise RstnetError(f"non-streaming forward_global over {T} > context = {self.config.context} positions is not "
                                  "implemented (the decode ring holds `context` keys); stream it instead")
            st = self._ns_state
            if st is None or st.B != B:
                st = self._ns_state = _LMState(self, B, parts=("temporal",))
            st.reset()
            return st.forward_global(sequence)
        return self._state.forward_global(sequence)

    @torch.no_grad()
    @on_own_device
    def forward_codecformer(self, codecformer_cb_index: int, sequence: torch.Tensor, transformer_out: torch.Tensor):
        B, K, S = sequence.shape
        assert K == 1, f"Codebooks for Depformer streaming should be passed 1 by 1, got {K}."
        assert S == 1, f"Steps for Depformer streaming should be passed 1 by 1, got {S}."
        assert transformer_out.shape[1] == 1, "Transformer out should be a for a single step."
        if self._state is None:
            raise RstnetError("forward_codecformer is the streaming form: call it inside `with gpt.streaming(B):` and "
                              "`with gpt.codecformer.streaming(B):` (forward_local is the non-streaming one)")
        return self._state.forward_codecformer(codecformer_cb_index, sequence, transformer_out)

    @torch.no_grad()
    @on_own_device
    def forward_local(self, local_start_token: torch.Tensor, sequence: torch.Tensor, transformer_out: torch.Tensor) -> torch.Tensor:
        """llama_streaming.py:694-725: the depth transformer over every (stream, frame) row, teacher-forced with
        `sequence[B, dep_q, T]`, non-streaming (every step sees all earlier keys).  -> logits [B, T, dep_q, card]."""
        self._check_runnable()
        c = self.config
        B, K, S = sequence.shape
        assert K == c.dep_q, f"Sequence shape {sequence.shape} must match the moshi stream output."
        rows = B * S
        start = local_start_token.reshape(rows, -1).to(torch.bfloat16)
        tout = transformer_out.reshape(rows, -1).to(torch.bfloat16)
        ids = sequence.permute(0, 2, 1).reshape(rows, K).to(torch.int64)
        out = torch.empty(rows, c.dep_q, c.audio_card, dtype=torch.bfloat16, device=self.device)
        for r0 in range(0, rows, MAX_ROWS):
            n = min(MAX_ROWS, rows - r0)
            self._depth_state(n).depth_local(start[r0:r0 + n], ids[r0:r0 + n], tout[r0:r0 + n], out[r0:r0 + n])
        return out.view(B, S, c.dep_q, c.audio_card)

    def _depth_state(self, n: int) -> "_LMState":
        """the depth-transformer-only state of n rows (forward_local, teacher-forced scoring)"""
        st = self._local_states.get(n)
        if st is None:
            if len(self._local_states) >= 4:
                self._local_states.clear()
            st = self._local_states[n] = _LMState(self, n, parts=("depth",))
        return st

    @torch.no_grad()
    @on_own_device
    def forward_step(self, sequence: torch.Tensor, *, use_sampling: bool = True, temp_text: float = 0.7, top_k_text: int = 25,
                     temp: float = 0.8, top_k: int = 30, audio_valid=2049, depth_ring_quirk: bool = True, sample_key=None,
                     sample_step=None) -> torch.Tensor:
        """One generated frame: temporal step on sequence[B,9,1], text token, then the 8 depth steps, each sampled
        on the device (sample_token / sample_token_audio[_2048], utils/sampling.py:85-154: use_sampling False ->
        argmax over the whole card; True -> temperature + top-k (top_k == 0: plain multinomial) over ids <
        audio_valid).  Returns tokens [B, 9] (text, audio_0..7).  With use_cuda_graphs the whole frame is a single
        graph replay.  depth_ring_quirk False evaluates the depth steps as forward_local does (see there).

        Per-row sampling (every row an utterance at its own point of generation): audio_valid as an int tensor
        [B, dep_q] gives each row its own candidate counts, and each row draws its noise from its own key and step
        counter instead of (row, scope frame counter).  sample_key [B] (uint32 values) and sample_step [B] (int64), when
        given, set the scope's per-row keys and step counters before the frame; otherwise they keep their values.  The
        step counters start at 0 (scope entry, reset_streaming of the row) and advance by one per frame for active rows.
        All three live in fixed device buffers, so one captured graph serves every frame."""
        if self._state is None:
            raise RstnetError("forward_step is a streaming call: use it inside `with gpt.streaming(B):`")
        return self._state.forward_step(sequence, use_sampling, temp_text, top_k_text, temp, top_k, audio_valid, depth_ring_quirk,
                                        sample_key, sample_step)

    @torch.no_grad()
    @on_own_device
    def prefill(self, sequence: torch.Tensor) -> None:
        """Feed sequence[B,9,T] through the temporal transformer (KV rings + positions advance by T) without producing
        outputs: what a prompt needs before generation starts (no lm_head, no depth steps)."""
        if self._state is None:
            raise RstnetError("prefill is a streaming call: use it inside `with gpt.streaming(B):`")
        self._state.forward_global(sequence, want_outputs=False)

    @torch.no_grad()
    @on_own_device
    def prefill_streams(self, prompts) -> None:
        """Feed each listed stream its own prompt: prompts {stream: int64 [9, T_s]}.  Stream s takes T_s positions from its
        current one on (KV ring + position counter, as prefill does for all streams); every other stream -- ring, position
        counter, active flag -- is left untouched, so utterances can join a scope while others are mid-generation.  The
        rows of all listed streams are packed into launches of at most MAX_ROWS rows."""
        if self._state is None:
            raise RstnetError("prefill_streams is a streaming call: use it inside `with gpt.streaming(B):`")
        self._state.prefill_streams(prompts)

    @torch.no_grad()
    @on_own_device
    def forward(self, sequence: torch.Tensor, input_pos: Optional[torch.Tensor] = None, lm_head_chunk_size: int = 0):
        """llama_streaming.py:651-663, the teacher-forced forward: the temporal transformer (non-streaming forward_global)
        over [initial token, sequence[:, :, :-1]], then the depth transformer (forward_local) started from the text
        embedding of each frame's own text token and fed sequence[:, 1:dep_q+1].  sequence [B, 9, S] ->
        (audio_logits [B, S, dep_q, card], text_logits [B, S, V]), bf16 (text_logits.squeeze(1) as upstream: [B, V] at S == 1).
        At most config.context frames (the existing limit of the non-streaming forward_global).  Evaluation only: no
        gradients.  lm_head_chunk_size is accepted and ignored, as upstream."""
        if self._state is not None:
            raise RstnetError("GPT.forward is the non-streaming teacher-forced form: call it outside `with gpt.streaming(B):`")
        if input_pos is not None:
            raise RstnetError("GPT.forward with input_pos (the KV-cache form) is not implemented; use gpt.streaming(B)")
        B, K, S = sequence.shape
        sequence = sequence.to(device=self.device, dtype=torch.int64)
        start = self._get_initial_token().repeat(B, 1, 1)
        transformer_out, text_logits = self.forward_global(torch.cat([start, sequence[:, :, :-1]], dim=2))
        text_logits = text_logits.squeeze(1)
        local_start = self.codecformer_text_emb(sequence[:, 0, :])
        audio_logits = self.forward_local(local_start, sequence[:, 1:self.config.dep_q + 1, :], transformer_out)
        return audio_logits, text_logits


# ------------------------------------------------------------------------------------------- teacher-forced scoring
CE_FIELDS = ("loss_sum", "count", "count_target", "correct", "correct_target")   # the 5 sums of one (slot, group)


def cross_entropy_sums(logits: torch.Tensor, labels: torch.Tensor, weights: torch.Tensor, groups: int,
                       ignore_ids: Optional[torch.Tensor] = None, row_slot: Optional[torch.Tensor] = None,
                       acc: Optional[torch.Tensor] = None, nll: Optional[torch.Tensor] = None,
                       pred: Optional[torch.Tensor] = None):
    """rstnet_lm_cross_entropy_bf16 on bf16 rows logits [rows, V] (last dim contiguous, any row stride): row i is group
    i % groups and slot row_slot[i] (None: slot 0).  labels int64 [rows], weights fp32 [rows], ignore_ids int64 [groups],
    all on the logits' device.  Adds into acc fp64 [slots, groups, 5] (see CE_FIELDS; allocated zero when None) and
    returns (acc, nll fp32 [rows], pred int32 [rows])."""
    if logits.device.type != "cuda" or logits.dtype != torch.bfloat16:
        raise RstnetError(f"the cross-entropy kernel reads bf16 logits on CUDA (got {logits.dtype} on {logits.device})")
    if logits.dim() != 2 or logits.stride(1) != 1:
        raise RstnetError("logits must be [rows, V] with contiguous rows")
    rows, V = logits.shape
    dev = logits.device
    n_slots = 1 if row_slot is None else (acc.shape[0] if acc is not None else int(row_slot.max()) + 1)
    for t, dt, n in ((labels, torch.int64, rows), (weights, torch.float32, rows)) + (
            ((row_slot, torch.int32, rows),) if row_slot is not None else ()) + (
            ((ignore_ids, torch.int64, groups),) if ignore_ids is not None else ()):
        if t.dtype != dt or t.device != dev or t.numel() != n or not t.is_contiguous():
            raise RstnetError(f"cross_entropy_sums: expected a contiguous {dt} tensor of {n} elements on {dev}")
    if acc is None:
        acc = torch.zeros(n_slots, groups, 5, dtype=torch.float64, device=dev)
    nll = torch.empty(rows, dtype=torch.float32, device=dev) if nll is None else nll
    pred = torch.empty(rows, dtype=torch.int32, device=dev) if pred is None else pred
    p = lambda t: None if t is None else t.data_ptr()
    _lib.check(_lib.lib().rstnet_lm_cross_entropy_bf16(logits.data_ptr(), logits.stride(0), rows, V, groups, labels.data_ptr(),
                                                       p(ignore_ids), weights.data_ptr(), p(row_slot), n_slots, nll.data_ptr(),
                                                       pred.data_ptr(), acc.data_ptr(), ops._stream()), "lm_cross_entropy")
    return acc, nll, pred


def combine_sums(sums, loss_weights) -> Dict[str, torch.Tensor]:
    """The host half of CrossEntropyAndAccuracy: sums [G, 5] (CE_FIELDS) -> loss = sum_g w_g * loss_sum_g / count_g (a group
    without a non-zero mask gives 0/0 = NaN, kept), acc_all / acc_target pooled over the groups.  fp64 scalars."""
    s = torch.as_tensor(sums, dtype=torch.float64).cpu().reshape(-1, 5)
    w = torch.as_tensor([float(x) for x in loss_weights], dtype=torch.float64)
    loss = (s[:, 0] / s[:, 1] * w).sum()
    return {"acc_all": s[:, 3].sum() / s[:, 1].sum(), "acc_target": s[:, 4].sum() / s[:, 2].sum(), "loss": loss}


def CrossEntropyAndAccuracy(logits, y, masks, loss_weights, ignore_ids=None):
    """models/model.py:31-65 on bf16 logits [B, T, G, V] (CUDA): labels y [B, G, T], masks [B, G, T] (float weights: loss
    rows are multiplied by them, `!= 0` and `== 1` select the counted tokens), one loss weight and ignore id per group.
    -> (loss, {'acc_all', 'acc_target', 'loss'}) as 0-dim fp64 tensors.  The per-row losses are fp32 and the sums fp64
    (upstream: bf16 rows).  A label outside [0, V) that is not its group's ignore id raises IndexError, as F.cross_entropy."""
    if logits.dim() != 4:
        raise RstnetError(f"logits must be [B, T, G, V], got {tuple(logits.shape)}")
    B, T, G, V = logits.shape
    dev = logits.device
    y, masks = torch.as_tensor(y).to(dev), torch.as_tensor(masks).to(dev)
    if tuple(y.shape) != (B, G, T) or tuple(masks.shape) != (B, G, T):
        raise RstnetError(f"labels and masks must be [B, G, T] = {(B, G, T)}, got {tuple(y.shape)} and {tuple(masks.shape)}")
    if len(loss_weights) != G:
        raise RstnetError(f"{len(loss_weights)} loss weights for {G} groups")
    if ignore_ids is not None and len(ignore_ids) != G:
        raise RstnetError(f"{len(ignore_ids)} ignore ids for {G} groups")
    try:
        rows = logits.view(B * T * G, V)
    except RuntimeError:
        rows = logits.contiguous().view(B * T * G, V)
    labels = y.permute(0, 2, 1).reshape(-1).to(torch.int64).contiguous()
    weights = masks.permute(0, 2, 1).reshape(-1).to(torch.float32).contiguous()
    ign = None if ignore_ids is None else torch.as_tensor([int(i) for i in ignore_ids], dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        acc, _, _ = cross_entropy_sums(rows, labels, weights, G, ign)
        flags = int(_lib.lib().rstnet_device_error_flags(1))
    if flags & 1:
        raise IndexError("a label was outside [0, V) and not its group's ignore id (Target out of bounds)")
    m = combine_sums(acc[0], loss_weights)
    return m["loss"], m


class _LMState:
    """Buffers, KV rings, GEMM plans of one `streaming(B)` scope.  Rows of every activation buffer are (position,
    stream) pairs, position-major: row = tl * B + b.  The decode state has tn == 1; a prefill chunk state (`parent` set)
    has tn > 1 rows per stream and shares the parent's KV rings and position counters; a `parts == ("depth",)` state
    only holds the depth transformer (forward_local)."""

    def __init__(self, m: GPT, B: int, tn: int = 1, parent: Optional["_LMState"] = None, parts=("temporal", "depth"),
                 rows: Optional[int] = None):
        """rows: a ragged prefill chunk of that many rows (with `parent`): row r is stream row_stream[r] at position
        offset + row_tl[r] (-1: padding), and the counters advance by `delta` per stream."""
        c, dev = m.config, m.device
        self.m, self.B, self.c, self.tn = m, B, c, tn
        M = self.M = B * tn if rows is None else rows
        if rows is not None and (parent is None or rows > MAX_ROWS):
            raise RstnetError(f"a ragged prefill chunk has a parent scope and at most {MAX_ROWS} rows (got {rows})")
        if tn == 1 and B > MAX_STREAMS:
            raise RstnetError(f"at most {MAX_STREAMS} streams per streaming scope (got {B})")
        if tn > 1 and M > MAX_ROWS:
            raise RstnetError(f"at most {MAX_ROWS} rows per launch sequence (got {B} streams x {tn} positions)")
        bf = torch.bfloat16
        P = {k: v for k, v in m.named_parameters()}
        E, V, I, D, H = c.n_embd, c.padded_vocab_size, c.intermediate_size, c.codecformer_dim, c.ff_hidden
        nh, nkv, hs = c.n_head, c.n_query_groups, c.head_size
        self.cap = c.context
        Hp = -(-H // 64) * 64  # the GEMMs' K granularity: pad the gating hidden size with zero weights
        self.Hp = Hp

        def z(*shape, dtype=bf):
            return torch.zeros(*shape, dtype=dtype, device=dev)

        if m._packed is None:
            pk = self._pack_temporal(P)
            # depth gating weights: K padded to the GEMM granularity.  They keep the stacked [gate; value] form + finalize
            # kernel: with 44 column tiles the GEMM's split-K heuristic picks two K slices, which the in-epilogue gating
            # cannot have.
            for l in range(c.codecformer_layers if Hp != H else 0):
                for k in range(c.dep_q):
                    w_in = P[m._DN["dlayer"].format(l) + f".gating.{k}.linear_in.weight"]
                    w_out = P[m._DN["dlayer"].format(l) + f".gating.{k}.linear_out.weight"]
                    gi = z(2 * Hp, D)
                    gi[:H], gi[Hp:Hp + H] = w_in[:H], w_in[H:]
                    go = z(D, Hp)
                    go[:, :H] = w_out
                    pk[f"gin.{l}.{k}"], pk[f"gout.{l}.{k}"] = gi, go
            m._packed = pk
        wsmax = max((nh + 2 * nkv) * hs, 2 * I, 4096, 3 * D, 2 * Hp)
        self.ws = parent.ws if parent is not None and parent.M >= M else torch.empty(8 * M * wsmax, dtype=torch.float32, device=dev)
        G = lambda X, W, out, R=None, **kw: SkinnyGemm(X, W, out, R, self.ws if W.shape[0] <= wsmax else None, **kw)
        self.graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self.warm: Dict[tuple, int] = {}
        self.seed = 1234
        self.depth_step: Optional[int] = None
        self.children: Dict[int, "_LMState"] = {}
        self.row_children: Dict[int, "_LMState"] = {}
        self.has_temporal = "temporal" in parts
        self.row_mapped = rows is not None
        if self.row_mapped:
            self.row_stream, self.row_tl = z(M, dtype=torch.int32), z(M, dtype=torch.int32)
            self.delta = z(B, dtype=torch.int64)

        if self.has_temporal:
            self._build_temporal(P, G, z, parent)

        if "depth" in parts:
            self.tout = z(M, E)
            self.demb, self.dx, self.dn, self.datt = z(M, D), z(M, D), z(M, D), z(M, D)
            self.dqkv, self.dh, self.dlogits = z(M, 3 * D), z(M, Hp), z(M, c.audio_card)
            self.tokens = z(M, c.dep_q + 1, dtype=torch.int64)
            self._idbuf = z(M, dtype=torch.int64)
            self.frame_counter = z(1, dtype=torch.int64)
            # per-row sampling (forward_step with an audio_valid table): candidate counts, RNG keys, step counters
            self.row_valid = z(M, c.dep_q, dtype=torch.int32)
            self.row_key = z(M, dtype=torch.int32)
            self.row_step = z(M, dtype=torch.int64)
            hd = D // c.codecformer_heads
            self.dkv_all = z(c.codecformer_layers, 2, M, c.codecformer_heads, c.dep_q, hd)
            self.dkv = [self.dkv_all[l] for l in range(c.codecformer_layers)]
            # depth transformer: per-codebook-step weight slabs
            DN = m._DN
            self.text_emb = P[DN["dtext"]]
            self.dep_emb = [P[DN["demb"].format(i)] for i in range(c.dep_q - 1)]
            Ld = c.codecformer_layers
            a1 = [P[DN["dlayer"].format(l) + ".norm1.alpha"].view(-1) for l in range(Ld)]
            a2 = [P[DN["dlayer"].format(l) + ".norm2.alpha"].view(-1) for l in range(Ld)]
            self.dsteps = []
            for k in range(c.dep_q):
                layers = []
                for l in range(Ld):
                    p = DN["dlayer"].format(l)
                    w_in = P[f"{p}.self_attn.in_proj_weight"].view(c.dep_q, 3 * D, D)[k]
                    w_out = P[f"{p}.self_attn.out_proj.weight"].view(c.dep_q, D, D)[k]
                    g_in = m._packed.get(f"gin.{l}.{k}", P[f"{p}.gating.{k}.linear_in.weight"])
                    g_out = m._packed.get(f"gout.{l}.{k}", P[f"{p}.gating.{k}.linear_out.weight"])
                    nxt = dict(norm_w=a1[l + 1], aux=self.dn, eps=1e-8, kyutai=True) if l + 1 < Ld else {}
                    layers.append(dict(
                        qkv=G(self.dn, w_in, self.dqkv),
                        out=G(self.datt, w_out, self.dx, self.dx, norm_w=a2[l], aux=self.dn, eps=1e-8, kyutai=True),
                        gin=G(self.dn, g_in, None, silu_out=self.dh),
                        gout=G(self.dh, g_out, self.dx, self.dx, **nxt)))
                self.dsteps.append(dict(
                    inp=G(self.tout, P[DN["din"].format(k)], self.dx, self.demb, norm_w=a1[0], aux=self.dn, eps=1e-8, kyutai=True),
                    layers=layers, head=G(self.dx, P[DN["dhead"].format(k)], self.dlogits)))

    def _pack_temporal(self, P):
        """one-time repacked weights of the temporal transformer (fc_1 and fc_2 interleaved as one GEMM)"""
        c = self.c
        return {f"fc12.{l}": interleave_gate_rows(P[f"transformer.h.{l}.mlp.fc_1.linear.weight"],
                                                  P[f"transformer.h.{l}.mlp.fc_2.linear.weight"])
                for l in range(c.n_layer)}

    def _build_temporal(self, P, G, z, parent):
        m, c, B, M = self.m, self.c, self.B, self.M
        dev, bf = m.device, torch.bfloat16
        E, V, I = c.n_embd, c.padded_vocab_size, c.intermediate_size
        nh, nkv, hs = c.n_head, c.n_query_groups, c.head_size
        self.seq = z(M, c.n_q + 1, dtype=torch.int64)
        self.x, self.xn, self.q, self.att = z(M, E), z(M, E), z(M, nh * hs), z(M, nh * hs)
        self.qkv, self.hmid = z(M, (nh + 2 * nkv) * hs), z(M, I)
        self.out, self.logits = z(M, E), z(M, V)
        if parent is None:
            # one position counter per stream (per-stream reset / admission), mirrored on the host for the
            # block_size check (under graph replay the device cannot raise)
            self.offset = z(B, dtype=torch.int64)
            self.pos_host = np.zeros(B, dtype=np.int64)
            # advance flags: a stream with 0 is HELD by the next steps (frame scheduler rows without input)
            self.active = torch.ones(B, dtype=torch.int64, device=dev)
            self.active_host = np.ones(B, dtype=np.int64)
            # KV rings, one K/V row per KV GROUP: [2, B, n_kv, cap, hs] (lit_model.py:607-615 stores n_head copies)
            self.kv = [z(2, B, nkv, self.cap, hs) for _ in range(c.n_layer)]
            # RoPE tables in the model dtype (the reference's buffers are cast by .to(bfloat16)); lit_model.py:441-488
            n = c.rope_n_elem
            theta = 1.0 / (c.rope_base ** (torch.arange(0, n, 2).float() / n))
            if c.rope_adjustments is not None:
                ec = c.rope_adjustments
                wavelen = 2 * torch.pi / theta
                ratio = ec["original_max_seq_len"] / wavelen
                smooth = torch.clamp((ratio - ec["low_freq_factor"]) / (ec["high_freq_factor"] - ec["low_freq_factor"]), min=0.0, max=1.0)
                theta = (1 - smooth) * (theta / ec["factor"]) + smooth * theta
            idx_theta = torch.outer(torch.arange(c.block_size) / c.rope_condense_ratio, theta).repeat(1, 2)
            self.cos, self.sin = torch.cos(idx_theta).to(bf).to(dev).contiguous(), torch.sin(idx_theta).to(bf).to(dev).contiguous()
        else:
            self.offset, self.pos_host, self.kv, self.cos, self.sin = parent.offset, parent.pos_host, parent.kv, parent.cos, parent.sin
            self.active, self.active_host = parent.active, parent.active_host
        self.tables = [P[f"input_emb.{i}.weight"] for i in range(c.n_q)]
        self.table_ptrs = torch.tensor([t.data_ptr() for t in self.tables], dtype=torch.int64, device=dev)
        self.wte = P["transformer.wte.weight"]
        L_ = c.n_layer
        n1 = [P[f"transformer.h.{l}.norm_1.weight"] for l in range(L_)]
        n2 = [P[f"transformer.h.{l}.norm_2.weight"] for l in range(L_)]
        self.ln_f = P["transformer.ln_f.weight"]
        self.n1_first = n1[0]
        self.layers = []
        for l in range(L_):
            p = f"transformer.h.{l}"
            last = l == L_ - 1
            self.layers.append(dict(
                qkv=G(self.xn, P[f"{p}.attn.attn.linear.weight"], self.qkv),
                # x = attn + x ; xn = norm_2(x)   (Block.forward, llama_streaming.py:846-849) in the GEMM's finalize
                proj=G(self.att, P[f"{p}.attn.proj.linear.weight"], self.x, self.x, norm_w=n2[l], aux=self.xn, eps=c.norm_eps),
                # hmid = silu(fc_1 x) * fc_2 x   (LLaMAMLP, lit_model.py:399-403)
                fc=G(self.xn, m._packed[f"fc12.{l}"], None, silu_out=self.hmid, interleaved=True),
                # x = mlp + x ; xn = norm_1 of the next block (or ln_f -> transformer_out)
                down=G(self.hmid, P[f"{p}.mlp.proj.linear.weight"], self.x, self.x, norm_w=self.ln_f if last else n1[l + 1],
                       aux=self.out if last else self.xn, eps=c.norm_eps)))
        self.head = G(self.out, P["lm_head.linear.weight"], self.logits)

    def reset(self, streams=None):
        if streams is None:
            self.offset.zero_()
            self.pos_host[:] = 0
        else:
            idx = torch.as_tensor(streams, dtype=torch.int64).reshape(-1)
            if idx.numel() and (int(idx.min()) < 0 or int(idx.max()) >= self.B):
                raise RstnetError(f"stream index outside [0, {self.B})")
            self.offset[idx.to(self.offset.device)] = 0
            self.pos_host[idx.numpy()] = 0
        if hasattr(self, "frame_counter"):
            self.frame_counter.zero_()
            if streams is None:
                self.row_step.zero_()
            else:
                self.row_step[idx.to(self.row_step.device)] = 0
        self.depth_step = None

    # ---- launch sequences -------------------------------------------------------------------
    def _temporal(self, head: bool = True):
        c, B, M, L = self.c, self.B, self.M, _lib.lib()
        st = ops._stream()
        E = c.n_embd
        ost = 1 if self.offset.numel() > 1 else 0
        _lib.check(L.rstnet_lm_embed_sum_bf16(self.seq.data_ptr(), c.n_q + 1, self.wte.data_ptr(), self.wte.shape[0],
                                              self.table_ptrs.data_ptr(), self.tables[0].shape[0], c.n_q, E, self.x.data_ptr(), M, st),
                   "lm_embed_sum")
        _lib.check(L.rstnet_lm_rms_norm_bf16(self.x.data_ptr(), self.n1_first.data_ptr(), self.xn.data_ptr(), M, E, c.norm_eps, 0, st), "rms")
        for l, ly in enumerate(self.layers):
            ly["qkv"].run()
            if self.row_mapped:
                _lib.check(L.rstnet_lm_rope_kv_append_rows_bf16(self.qkv.data_ptr(), self.cos.data_ptr(), self.sin.data_ptr(),
                                                                self.cos.shape[0], c.rope_n_elem, self.offset.data_ptr(),
                                                                self.row_stream.data_ptr(), self.row_tl.data_ptr(), self.q.data_ptr(),
                                                                self.kv[l].data_ptr(), M, B, c.n_head, c.n_query_groups,
                                                                c.head_size, self.cap, st), "rope_kv_rows")
                _lib.check(L.rstnet_lm_ring_decode_attention_rows_bf16(self.q.data_ptr(), self.kv[l].data_ptr(), self.offset.data_ptr(),
                                                                       self.row_stream.data_ptr(), self.row_tl.data_ptr(),
                                                                       self.att.data_ptr(), M, B, c.n_head, c.n_query_groups,
                                                                       c.head_size, self.cap, c.context, st), "attention_rows")
                ly["proj"].run()
                ly["fc"].run()
                ly["down"].run()
                continue
            _lib.check(L.rstnet_lm_rope_kv_append_bf16(self.qkv.data_ptr(), self.cos.data_ptr(), self.sin.data_ptr(), self.cos.shape[0],
                                                       c.rope_n_elem, self.offset.data_ptr(), ost, self.q.data_ptr(),
                                                       self.kv[l].data_ptr(), M, B, c.n_head, c.n_query_groups, c.head_size, self.cap, st),
                       "rope_kv")
            _lib.check(L.rstnet_lm_ring_decode_attention_bf16(self.q.data_ptr(), self.kv[l].data_ptr(), self.offset.data_ptr(), ost,
                                                              self.att.data_ptr(), M, B, c.n_head, c.n_query_groups, c.head_size,
                                                              self.cap, c.context, st), "attention")
            ly["proj"].run()   # + residual + norm_2 -> xn
            ly["fc"].run()     # + SiLU gating -> hmid
            ly["down"].run()   # + residual + next pre-norm -> xn (last layer: ln_f -> transformer_out)
        if head:
            self.head.run()
        if self.row_mapped:
            _lib.check(L.rstnet_counter_add_rows(self.offset.data_ptr(), self.delta.data_ptr(), B, st), "counter_add_rows")
        else:
            ops.counter_add(self.offset, self.tn, self.active)

    def _depth(self, k: int, ids: Optional[torch.Tensor], id_stride: int, quirk: bool = True):
        """ids None: the step's input embedding is already in self.demb (forward_local passes features for step 0)."""
        c, M, L = self.c, self.M, _lib.lib()
        st = ops._stream()
        D = c.codecformer_dim
        if ids is not None:
            table = self.text_emb if k == 0 else self.dep_emb[k - 1]
            _lib.check(L.rstnet_lm_embed_rows_bf16(ids.data_ptr(), id_stride, table.data_ptr(), table.shape[0], D, self.demb.data_ptr(), M, st),
                       "embed_rows")
        ds = self.dsteps[k]
        ds["inp"].run()        # dx = in_k(transformer_out) + emb ; dn = norm1_0(dx)
        hd = D // c.codecformer_heads
        for l, ly in enumerate(ds["layers"]):
            ly["qkv"].run()
            _lib.check(L.rstnet_lm_depth_attention_bf16(self.dqkv.data_ptr(), self.dkv[l].data_ptr(), self.datt.data_ptr(), M,
                                                        c.codecformer_heads, hd, c.dep_q, k, int(quirk), st), "depth_attention")
            ly["out"].run()    # dx += out_k(att) ; dn = norm2(dx)
            ly["gin"].run()    # dh = silu(a) * b
            ly["gout"].run()   # dx += out(dh) ; dn = norm1 of the next layer
        ds["head"].run()

    def _sample(self, logits: torch.Tensor, V: int, n_valid: int, top_k: int, temp: float, col: int, salt: int):
        _lib.check(_lib.lib().rstnet_lm_sample_bf16(logits.data_ptr(), self.M, V, n_valid, top_k, float(temp), self.seed + salt,
                                                    self.frame_counter.data_ptr(), self.tokens.data_ptr() + 8 * col,
                                                    self.c.dep_q + 1, ops._stream()), "sample")

    def _sample_rows(self, logits: torch.Tensor, V: int, per_row_valid: Optional[int], top_k: int, temp: float, col: int, salt: int):
        """per_row_valid: column of row_valid holding the rows' candidate counts (None: all V ids)"""
        nv = None if per_row_valid is None else self.row_valid.data_ptr() + 4 * per_row_valid
        _lib.check(_lib.lib().rstnet_lm_sample_rows_bf16(logits.data_ptr(), self.M, V, V, nv, self.c.dep_q, top_k, float(temp),
                                                         self.seed + salt, self.row_step.data_ptr(), self.row_key.data_ptr(),
                                                         self.tokens.data_ptr() + 8 * col, self.c.dep_q + 1, ops._stream()),
                   "sample_rows")

    def _replay(self, key, fn):
        if not self.m.use_cuda_graphs:
            fn()
            return
        g = self.graphs.get(key)
        if g is None:
            self.warm[key] = self.warm.get(key, 0) + 1
            if self.warm[key] <= 1:
                fn()
                return
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                fn()
            self.graphs[key] = g
        g.replay()

    def _advance_host(self, n: int):
        """Host mirror of the position counters: the reference's cos.index_select raises past block_size
        (llama_streaming.py:972-975); a graph replay cannot, so the check happens here, before the launch."""
        if int(self.pos_host.max()) + n > self.cos.shape[0]:
            raise IndexError(f"position {int(self.pos_host.max()) + n - 1} is beyond block_size = {self.cos.shape[0]} "
                             "(RoPE table exhausted; reset the stream or raise Config.block_size)")
        self.pos_host += n * self.active_host

    def set_active(self, mask):
        """mask [B]: streams with 0 are held by the next steps (they run through the kernels, but their position does not
        advance; the K/V row written at the held position is overwritten by the stream's next real step)."""
        if mask is None:
            self.active.fill_(1)
            self.active_host[:] = 1
        else:
            mk = torch.as_tensor(mask).to(dtype=torch.int64).reshape(self.B).cpu()
            self.active_host[:] = mk.numpy()
            self.active.copy_(mk.to(self.active.device))

    # ---- API ----------------------------------------------------------------------------------
    def forward_global(self, sequence: torch.Tensor, want_outputs: bool = True):
        c = self.c
        B, K, T = sequence.shape
        if B != self.B:
            raise RstnetError(f"streaming batch size is {self.B}, got {B}")
        if T == 1:
            self._advance_host(1)
            self.seq.copy_(sequence[:, :, 0])
            if want_outputs:
                self._replay(("temporal",), self._temporal)
                return self.out.view(B, 1, c.n_embd).clone(), self.logits.view(B, 1, c.padded_vocab_size).clone()
            self._replay(("temporal_nohead",), lambda: self._temporal(head=False))
            return None
        # prefill: chunks of tn consecutive positions for all streams (tn * B <= MAX_ROWS rows per launch sequence; more
        # than MAX_ROWS streams go one position per pass through the decode state).
        # A multi-position chunk appends all its keys before any of its queries run, so it must not overwrite a ring slot
        # one of those queries still needs: tn > 1 only while the ring does not wrap inside the chunk.
        outs, logits = [], []
        per = max(1, MAX_ROWS // B)
        t = 0
        while t < T:
            tn = min(per, T - t)
            if tn > 1 and int(self.pos_host.max()) + tn > self.cap:
                tn = 1
            if tn == 1:
                r = self.forward_global(sequence[:, :, t:t + 1], want_outputs)
                if want_outputs:
                    outs.append(r[0]); logits.append(r[1])
            else:
                ch = self.children.get(tn)
                if ch is None:
                    if len(self.children) >= 2:      # keep at most two chunk shapes alive (full chunk + one tail)
                        self.children.pop(next(iter(self.children)))
                    ch = self.children[tn] = _LMState(self.m, B, tn=tn, parent=self, parts=("temporal",))
                self._advance_host(tn)
                ch.seq.copy_(sequence[:, :, t:t + tn].permute(2, 0, 1).reshape(tn * B, K))
                ch._temporal(head=want_outputs)
                if want_outputs:
                    outs.append(ch.out.view(tn, B, c.n_embd).permute(1, 0, 2).clone())
                    logits.append(ch.logits.view(tn, B, c.padded_vocab_size).permute(1, 0, 2).clone())
            t += tn
        if not want_outputs:
            return None
        return torch.cat(outs, 1), torch.cat(logits, 1)

    def prefill_streams(self, prompts):
        c, dev = self.c, self.m.device
        K = c.n_q + 1
        todo = []   # [stream, prompt [T, K] on the device, positions fed]
        for s, p in prompts.items():
            s = int(s)
            if not 0 <= s < self.B:
                raise RstnetError(f"stream index {s} outside [0, {self.B})")
            if p.dim() != 2 or p.shape[0] != K:
                raise RstnetError(f"the prompt of stream {s} must be [{K}, T], got {tuple(p.shape)}")
            if p.shape[1] > self.m.max_seq_length:
                raise ValueError(f"Cannot forward sequence of length {p.shape[1]}, max seq length is only {self.m.max_seq_length}.")
            if int(self.pos_host[s]) + p.shape[1] > self.cos.shape[0]:
                raise IndexError(f"position {int(self.pos_host[s]) + p.shape[1] - 1} of stream {s} is beyond block_size = "
                                 f"{self.cos.shape[0]} (RoPE table exhausted; reset the stream or raise Config.block_size)")
            if p.shape[1] > 0:
                todo.append([s, p.to(device=dev, dtype=torch.int64).t(), 0])
        while todo:
            self.row_chunk(todo)
            todo = [it for it in todo if it[2] < it[1].shape[0]]

    def row_chunk(self, todo, head: bool = False):
        """One launch sequence of a ragged prefill: rows of the [stream, feed [T, K] on the device, positions fed] entries
        of `todo`, in order, up to MAX_ROWS; advances each entry's count and its stream's position.  head: also run the
        lm_head.  -> (chunk state, [(stream, first row, first position fed, positions)] per stream in the chunk); the
        chunk's out / logits rows are valid until the next chunk of the same width."""
        c, dev = self.c, self.m.device
        K = c.n_q + 1
        rs, rt, parts, segs = [], [], [], []
        delta = np.zeros(self.B, dtype=np.int64)
        for it in todo:
            s, p, done = it
            budget = MAX_ROWS - len(rs)
            if budget == 0:
                break
            if done >= p.shape[0]:
                continue
            # a chunk appends all its keys before any of its queries run: several positions of a stream only while its
            # ring does not wrap inside the chunk (as forward_global's prefill), one per chunk after that
            tn = min(p.shape[0] - done, budget, max(1, self.cap - int(self.pos_host[s])))
            segs.append((s, len(rs), done, tn))
            rs += [s] * tn
            rt += range(tn)
            parts.append(p[done:done + tn])
            delta[s] = tn
            it[2] += tn
        n = len(rs)
        M = next(b for b in ROW_BUCKETS if b >= n)
        ch = self.row_children.get(M)
        if ch is None:
            ch = self.row_children[M] = _LMState(self.m, self.B, parent=self, parts=("temporal",), rows=M)
        pad = M - n
        ch.row_stream.copy_(torch.tensor(rs + [-1] * pad, dtype=torch.int32))
        ch.row_tl.copy_(torch.tensor(rt + [0] * pad, dtype=torch.int32))
        ch.delta.copy_(torch.from_numpy(delta))
        if pad:
            parts.append(torch.full((pad, K), self.m.zero_token_id, dtype=torch.int64, device=dev))   # an all-zero-token row
        ch.seq.copy_(torch.cat(parts))
        ch._temporal(head=head)
        self.pos_host += delta
        return ch, segs

    def forward_codecformer(self, k: int, sequence: torch.Tensor, transformer_out: torch.Tensor):
        if self.depth_step is None:
            raise RstnetError("call inside `with gpt.codecformer.streaming(B):`")
        if k != self.depth_step:
            raise RstnetError(f"depth steps must run in order: expected {self.depth_step}, got {k}")
        self.tout.copy_(transformer_out[:, 0])
        self._idbuf.copy_(sequence[:, 0, 0])
        self._replay(("depth", k), lambda: self._depth(k, self._idbuf, 1))
        self.depth_step += 1
        return self.dlogits.view(self.B, 1, 1, self.c.audio_card).clone()

    def depth_local(self, start: torch.Tensor, ids: torch.Tensor, tout: torch.Tensor, out: torch.Tensor):
        """forward_local on self.M rows: start [M, D] features of step 0, ids [M, dep_q] teacher-forced tokens
        (column k-1 feeds step k), tout [M, E]; writes out [M, dep_q, card]."""
        c = self.c
        self.tout.copy_(tout)
        self.tokens[:, :c.dep_q].copy_(ids)
        for k in range(c.dep_q):
            if k == 0:
                self.demb.copy_(start)
                self._depth(0, None, 0, quirk=False)
            else:
                self._depth(k, self.tokens[:, k - 1], c.dep_q + 1, quirk=False)
            out[:, k].copy_(self.dlogits)

    def depth_teacher(self, tout: torch.Tensor, frames: torch.Tensor, out: torch.Tensor):
        """forward_local on self.M rows whose step-0 feature is the embedding of the row's own text token (GPT.forward):
        frames int64 [M, dep_q + 1] = (text, audio_0 .. audio_{dep_q-1}) of each row, tout [M, E]; writes out
        [M, dep_q, card].  The text embedding is the bounds-checked gather of the decode step, not a host-side lookup."""
        c = self.c
        self.tout.copy_(tout)
        self.tokens.copy_(frames)
        for k in range(c.dep_q):
            self._depth(k, self.tokens[:, k], c.dep_q + 1, quirk=False)
            out[:, k].copy_(self.dlogits)

    def forward_step(self, sequence, use_sampling, temp_text, top_k_text, temp, top_k, audio_valid, quirk=True, sample_key=None,
                     sample_step=None):
        c = self.c
        if sequence.shape[0] != self.B or sequence.shape[2] != 1:
            raise RstnetError(f"forward_step takes sequence [{self.B}, {c.n_q + 1}, 1], got {tuple(sequence.shape)}")
        per_row = torch.is_tensor(audio_valid)
        if per_row:
            if tuple(audio_valid.shape) != (self.B, c.dep_q):
                raise RstnetError(f"a per-row audio_valid is [{self.B}, {c.dep_q}], got {tuple(audio_valid.shape)}")
            if sample_key is not None:
                k = torch.as_tensor(sample_key, dtype=torch.int64).reshape(self.B) & 0xFFFFFFFF
                self.row_key.copy_(torch.where(k >= 2 ** 31, k - 2 ** 32, k).to(torch.int32))   # the uint32 bits
            if sample_step is not None:
                self.row_step.copy_(torch.as_tensor(sample_step, dtype=torch.int64).reshape(self.B))
        elif sample_key is not None or sample_step is not None:
            raise RstnetError("sample_key / sample_step select per-row sampling: pass audio_valid as a [B, dep_q] tensor")
        self._advance_host(1)
        self.seq.copy_(sequence[:, :, 0])
        if per_row:
            self.row_valid.copy_(audio_valid)
            self._replay(*self._frame_rows(use_sampling, temp_text, top_k_text, temp, top_k, quirk))
        else:
            self._replay(*self._frame(use_sampling, temp_text, top_k_text, temp, top_k, audio_valid, quirk))
        return self.tokens.clone()

    def _frame_rows(self, use_sampling, temp_text, top_k_text, temp, top_k, quirk):
        """_frame with per-row candidate counts (row_valid), RNG keys (row_key) and step counters (row_step)."""
        c = self.c
        sampling_text = use_sampling and temp_text > 0.0
        sampling = use_sampling and temp > 0.0
        tk_text = (top_k_text if top_k_text > 0 else -1) if sampling_text else 0
        tk = (top_k if top_k > 0 else -1) if sampling else 0

        def frame():
            self._temporal()
            self._sample_rows(self.logits, c.padded_vocab_size, None, tk_text, temp_text if sampling_text else 1.0, 0, 0)
            self.tout.copy_(self.out)
            for k in range(c.dep_q):
                self._depth(k, self.tokens[:, k], c.dep_q + 1, quirk=quirk)
                # the 2048 / 2049 candidate sets exist on the sampling path only (sampling.py:107-154)
                self._sample_rows(self.dlogits, c.audio_card, k if sampling else None, tk, temp if sampling else 1.0, k + 1, k + 1)
            ops.counter_add(self.row_step, 1, self.active)

        return ("frame_rows", tk_text, float(temp_text), tk, float(temp), bool(quirk)), frame

    def _frame(self, use_sampling, temp_text, top_k_text, temp, top_k, audio_valid, quirk):
        """(graph key, launch sequence) of one generated frame from the ids in self.seq to the tokens in self.tokens."""
        c = self.c
        # kernel convention: 0 = argmax, k > 0 = top-k, -1 = multinomial over the whole (valid) support
        sampling_text = use_sampling and temp_text > 0.0
        sampling = use_sampling and temp > 0.0
        tk_text = (top_k_text if top_k_text > 0 else -1) if sampling_text else 0
        tk = (top_k if top_k > 0 else -1) if sampling else 0
        valid = tuple(audio_valid) if isinstance(audio_valid, (tuple, list)) else (audio_valid,) * c.dep_q
        if not sampling:
            valid = (c.audio_card,) * c.dep_q   # the 2048 / 2049 masks exist on the sampling path only (sampling.py:107-154)

        def frame():
            self._temporal()
            self._sample(self.logits, c.padded_vocab_size, c.padded_vocab_size, tk_text, temp_text if sampling_text else 1.0, 0, 0)
            self.tout.copy_(self.out)
            for k in range(c.dep_q):
                self._depth(k, self.tokens[:, k], c.dep_q + 1, quirk=quirk)
                self._sample(self.dlogits, c.audio_card, min(valid[k], c.audio_card), tk, temp if sampling else 1.0, k + 1, k + 1)
            ops.counter_add(self.frame_counter, 1)

        return ("frame", tk_text, float(temp_text), tk, float(temp), valid, bool(quirk)), frame
