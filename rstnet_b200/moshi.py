"""H100-native streaming decode path of the Moshi-style `LMModel` / `LMGen` twin of the reference.

Mirrors ``models.model.LMModel`` (MLLM_v2/models/model.py:98-428) and ``LMGen`` (:440-597) -- the model
`moshi/server.py:44-166` drives: a Kyutai `StreamingTransformer` backbone (rms_norm_f32, pair-RoPE, SiLU gating,
ring KV cache with `context` entries; modules/transformer.py) over the sum of n_q audio-codebook embeddings and a text
embedding, a text head, and the depth transformer with per-codebook-step weights.  Same constructor arguments, same
``state_dict`` keys, same streaming API:

  * ``LMModel.forward_text(sequence[B, K, 1]) -> (transformer_out[B,1,dim], text_logits[B,1,1,text_card])`` (:364-389)
  * ``with lm.depformer.streaming(B): lm.forward_depformer(k, prev[B,1,1], transformer_out) -> [B,1,1,card]`` (:392-428)
  * ``LMGen(lm, use_sampling, temp, temp_text, top_k, top_k_text).step(input_tokens[B, K_in, 1]) -> [B, dep_q+1, 1] | None``
    with the delay cache of :490-562 (acoustic delays, initial tokens, `max_delay` warm-up frames returning None).

Outside a streaming scope, the evaluation forward of the same file (:297-389): ``forward_text`` over whole sequences,
``forward_local`` and ``forward(sequence, masks) -> (audio_logits, text_logits)``, with the non-streaming attention
window of `context` positions at any length; ``score_many`` runs the reference trainer's `validate_model` over a corpus.

Extensions for serving a batch of sessions (rstnet_b200.serve.MoshiDuplexEngine): the delay cache keeps one step count per
row, so `LMGen.reset_streaming(streams=...)` restarts single rows and `LMGen.set_active_streams(mask)` holds rows, each
with its own warm-up (`LMGen.valid_rows()`).

The kernels are the GPT path's (rstnet_b200/lm.py): weight-streaming wgmma GEMMs with fused Kyutai RMSNorm / SiLU gating
finalizes, ring decode attention, the depth transformer, device-side sampling; plus the bf16 pair-RoPE kernel and the
two delay-cache kernels (csrc/delay_cache.cu).  One `LMGen.step` is one input copy and one CUDA-graph replay: cache_in,
the temporal step, text sampling, the dep_q depth steps with sampling, cache_out.
"""
from __future__ import annotations

import math
from contextlib import contextmanager
from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch
from torch import nn

from . import _lib, ops
from ._lib import RstnetError
from .codec import _register, on_own_device
from .lm import (KV_PAGE, MAX_ROWS, MAX_STREAMS, Sampling, _DecodeModel, _DepthScope, _LMState, _head_mode, combine_sums,
                 score_item, score_packed)


class _MoshiState(_LMState):
    """`_LMState` with the Kyutai temporal layer: in_proj (p h d) -> pair-RoPE -> ring attention -> out_proj, gating FFN."""

    kyutai_norm = 1

    def _pack_temporal(self, P):
        return {}

    def _build_temporal(self, P, G, z, parent):
        m, c = self.m, self.c
        dev, hs = m.device, c.head_size
        # freqs exactly as modules/rope.py:35-36 evaluates them (fp32 tensor * python scalar, then exp)
        ds = torch.arange(hs // 2, dtype=torch.float32)
        self.freqs = torch.exp(ds * (-math.log(m.max_period) * 2 / hs)).to(dev)
        self.tables = [P[f"emb.{i}.weight"] for i in range(c.n_q)]
        self.table_ptrs = torch.tensor([t.data_ptr() for t in self.tables], dtype=torch.int64, device=dev)
        self.wte = P["text_emb.weight"]
        L_ = c.n_layer
        a1 = [P[f"transformer.layers.{l}.norm1.alpha"].view(-1) for l in range(L_)]
        a2 = [P[f"transformer.layers.{l}.norm2.alpha"].view(-1) for l in range(L_)]
        self.n1_first = a1[0]
        out_norm = P["out_norm.alpha"].view(-1)
        kw = dict(eps=1e-8, kyutai=True)
        self.layers = []
        for l in range(L_):
            p = f"transformer.layers.{l}"
            last = l == L_ - 1
            self.layers.append(dict(
                qkv=G(self.xn, P[f"{p}.self_attn.in_proj_weight"], self.qkv),
                # x = x + out_proj(att) ; xn = norm2(x)      (_sa_block / _ff_block, modules/transformer.py:550-577)
                proj=G(self.att, P[f"{p}.self_attn.out_proj.weight"], self.x, self.x, norm_w=a2[l], aux=self.xn, **kw),
                # hmid = silu(a) * b with [a; b] = linear_in(xn)   (gating.py:12-21)
                fc=G(self.xn, P[f"{p}.gating.linear_in.weight"], None, silu_out=self.hmid),
                # x = x + linear_out(hmid) ; xn = norm1 of the next layer (last: out_norm -> transformer_out)
                down=G(self.hmid, P[f"{p}.gating.linear_out.weight"], self.x, self.x, norm_w=out_norm if last else a1[l + 1],
                       aux=self.out if last else self.xn, **kw)))
        self.head = G(self.out, P["text_linear.weight"], self.logits)

    def _offset_stride(self) -> int:
        return 1   # the pair-RoPE and attention launches index the counters per stream, even with B == 1

    def _rope_kv(self, L, l: int, ost: int, rs, rt, pg, st) -> None:
        """layer l's pair-RoPE at the positions' fp32 angles and the K/V append; a row-mapped chunk (row_chunk) runs a
        row-map entry point, the paged one on a paged scope"""
        c = self.c
        if self.row_mapped and self.pages is None:
            _lib.check(L.rstnet_lm_rope_pair_kv_append_rows_bf16(self.qkv.data_ptr(), self.offset.data_ptr(), rs, rt, self.q.data_ptr(),
                                                                 self.kv[l].data_ptr(), self.M, self.B, c.n_head, c.head_size, self.cap,
                                                                 self.freqs.data_ptr(), st), "rope_pair_kv_rows")
        elif self.row_mapped:
            _lib.check(L.rstnet_lm_rope_pair_kv_append_paged_rows_bf16(
                self.qkv.data_ptr(), self.offset.data_ptr(), rs, rt, self.q.data_ptr(), self.kv[l].data_ptr(), self.M, self.B, c.n_head,
                c.head_size, self.cap, self.freqs.data_ptr(), *pg, st), "rope_pair_kv_paged_rows")
        else:
            rope = L.rstnet_lm_rope_pair_kv_append_bf16 if self.pages is None else L.rstnet_lm_rope_pair_kv_append_paged_bf16
            _lib.check(rope(self.qkv.data_ptr(), self.offset.data_ptr(), ost, self.q.data_ptr(), self.kv[l].data_ptr(), self.M, self.B,
                            c.n_head, c.head_size, self.cap, self.freqs.data_ptr(), *pg, st), "rope_pair_kv")


class LMModel(_DecodeModel):
    """Drop-in for ``models.model.LMModel`` (same constructor arguments / defaults): the streaming decode path, and the
    non-streaming evaluation forward (forward_text over whole sequences, forward_local, forward)."""

    _DN = dict(din="depformer_in.{}.weight", demb="depformer_emb.{}.weight", dtext="depformer_text_emb.weight",
               dlayer="depformer_.layers.{}", dhead="linears.{}.weight")
    _RENAME = (("depformer_.", "depformer."),)

    def __init__(self, delays: List[int] = [0], n_q: int = 8, dep_q: int = 8, card: int = 1024, text_card: int = 32000, dim: int = 128,
                 num_heads: int = 8, hidden_scale: float = 4, norm: str = "layer_norm", norm_emb: bool = False, bias_proj: bool = False,
                 depformer_dim: int = 256, depformer_dim_feedforward=None, depformer_multi_linear: bool = False,
                 depformer_weights_per_step: bool = False, depformer_pos_emb: str = "sin", existing_text_padding_id: Optional[int] = None,
                 context: Optional[int] = None, device=None, dtype=None, **kwargs):
        super().__init__()
        num_layers = kwargs.get("num_layers", 6)
        dnl, dnh = kwargs.get("depformer_num_layers", num_layers), kwargs.get("depformer_num_heads", num_heads)
        unsupported = []
        if norm != "rms_norm_f32":
            unsupported.append(f"norm={norm!r} (rms_norm_f32 only)")
        if kwargs.get("gating", "none") != "silu" or kwargs.get("depformer_gating", kwargs.get("gating")) != "silu":
            unsupported.append("gating other than 'silu'")
        if kwargs.get("positional_embedding", "sin") != "rope" or depformer_pos_emb != "none":
            unsupported.append("positional embeddings other than rope (temporal) / none (depth)")
        if not (depformer_multi_linear and depformer_weights_per_step):
            unsupported.append("depformer without multi_linear / weights_per_step")
        if norm_emb or bias_proj or kwargs.get("layer_scale") is not None or not kwargs.get("causal", True) or context is None:
            unsupported.append("norm_emb / bias_proj / layer_scale / non-causal / context=None")
        if isinstance(depformer_dim_feedforward, (list, tuple)):
            unsupported.append("per-step depformer_dim_feedforward lists")
        if unsupported:
            raise NotImplementedError("LMModel here covers the configuration of moshi/models/loaders.py:68-98; unsupported: "
                                      + "; ".join(unsupported))
        self.n_q, self.dep_q, self.card, self.text_card, self.dim = n_q, dep_q, card, text_card, dim
        assert len(delays) == n_q + 1, "unexpected number of delays"
        self.delays = list(delays)
        self.existing_text_padding_id = existing_text_padding_id
        self.context = context
        self.max_period = float(kwargs.get("max_period", 10000))
        ff = int(hidden_scale * dim)
        hidden = (21 * dim) // 8 if ff == 4 * dim else (2 * ff) // 3          # modules/gating.py:40-43
        dff = int(hidden_scale * depformer_dim) if depformer_dim_feedforward is None else int(depformer_dim_feedforward)
        extra_text = existing_text_padding_id is None
        g = torch.Generator(device=device if device is not None else "cpu").manual_seed(0)
        fk = dict(device=device, dtype=dtype)
        w_ = lambda *shape: torch.empty(*shape, **fk).normal_(0.0, 0.02, generator=g)
        ones = lambda *shape: torch.ones(*shape, **fk)
        for i in range(n_q):
            _register(self, f"emb.{i}.weight", w_(card + 1, dim))
        _register(self, "text_emb.weight", w_(text_card + 1, dim))
        _register(self, "text_linear.weight", w_(text_card + extra_text, dim))
        for l in range(num_layers):
            p = f"transformer.layers.{l}"
            _register(self, f"{p}.self_attn.in_proj_weight", w_(3 * dim, dim))
            _register(self, f"{p}.self_attn.out_proj.weight", w_(dim, dim))
            _register(self, f"{p}.norm1.alpha", ones(1, 1, dim))
            _register(self, f"{p}.norm2.alpha", ones(1, 1, dim))
            _register(self, f"{p}.gating.linear_in.weight", w_(2 * hidden, dim))
            _register(self, f"{p}.gating.linear_out.weight", w_(dim, hidden))
        _register(self, "out_norm.alpha", ones(1, 1, dim))
        D = depformer_dim
        dh = (21 * D) // 8 if dff == 4 * D else (2 * dff) // 3
        for i in range(dep_q):
            _register(self, f"depformer_in.{i}.weight", w_(D, dim))
        for i in range(dep_q - 1):
            _register(self, f"depformer_emb.{i}.weight", w_(card + 1, D))
        _register(self, "depformer_text_emb.weight", w_(text_card + 1, D))
        for l in range(dnl):
            p = f"depformer_.layers.{l}"
            _register(self, f"{p}.self_attn.in_proj_weight", w_(dep_q * 3 * D, D))
            _register(self, f"{p}.self_attn.out_proj.weight", w_(dep_q * D, D))
            _register(self, f"{p}.norm1.alpha", ones(1, 1, D))
            _register(self, f"{p}.norm2.alpha", ones(1, 1, D))
            for k in range(dep_q):
                _register(self, f"{p}.gating.{k}.linear_in.weight", w_(2 * dh, D))
                _register(self, f"{p}.gating.{k}.linear_out.weight", w_(D, dh))
        for i in range(dep_q):
            _register(self, f"linears.{i}.weight", w_(card, D))
        # the fields `_LMState` reads, under the GPT config's names
        self.config = SimpleNamespace(n_embd=dim, padded_vocab_size=text_card + extra_text, intermediate_size=hidden, n_layer=num_layers,
                                      n_head=num_heads, n_query_groups=num_heads, head_size=dim // num_heads, context=context,
                                      n_q=n_q, dep_q=dep_q, audio_card=card, codecformer_dim=D, codecformer_heads=dnh,
                                      codecformer_layers=dnl, ff_hidden=dh, norm_eps=1e-8, block_size=1 << 62, rope_n_elem=0)
        self.depformer = _DepthScope(self)

    def _make_state(self, B: int, **kw) -> _MoshiState:
        return _MoshiState(self, B, **kw)

    def _scratch_state(self, B: int) -> _MoshiState:
        """A temporal scope of B streams for the non-streaming pass: rings of context + MAX_ROWS - 1 slots, so a chunk of up
        to MAX_ROWS consecutive positions never overwrites a key an earlier row of the same chunk still needs, and the
        window of `context` positions is exact at any length.  Attention runs with this cap and the model's context."""
        return _MoshiState(self, B, parts=("temporal",), cap=self.context + MAX_ROWS - 1)

    # ---- token conventions (models/model.py:226-288)
    @property
    def initial_token_id(self) -> int:
        return self.card

    @property
    def text_initial_token_id(self) -> int:
        return self.text_card

    @property
    def text_padding_token_id(self) -> int:
        return self.text_card if self.existing_text_padding_id is None else self.existing_text_padding_id

    @property
    def end_of_text_padding_id(self) -> int:
        return 0

    def _st(self) -> _MoshiState:
        if self._state is None:
            raise RstnetError("only the streaming decode path is implemented: call inside `with lm.streaming(B):`")
        return self._state

    # ---- reference API
    @torch.no_grad()
    @on_own_device
    def forward_text(self, sequence: torch.Tensor):
        """models/model.py:364-389.  Inside a streaming scope: one frame per call (the decode step).  Outside: the
        non-streaming form over positions 0..S-1 from scratch, nothing kept, each position attending over the last
        `context` positions (modules/transformer.py:399-405) at any S.  -> (transformer_out [B, S, dim], text_logits
        [B, 1, S, text_card]), bf16."""
        B, K, S = sequence.shape
        assert K == self.num_codebooks, f"Sequence shape {sequence.shape} must match the number of codebooks."
        if self._state is None:
            self._check_runnable()
            st = self._ns_state
            if st is None or st.B != B:
                self._ns_state = None                    # free the old rings before the new ones are allocated
                st = self._ns_state = self._scratch_state(B)
            st.reset()
            out, logits = st.forward_global(sequence.to(device=self.device, dtype=torch.int64))
            return out, logits[:, None]
        if S != 1:
            raise RstnetError("streaming forward_text takes one frame per call")
        out, logits = self._st().forward_global(sequence)
        return out, logits[:, None]                                  # [B,1,dim], [B,1,1,text_card]

    @torch.no_grad()
    @on_own_device
    def prefill_streams(self, feeds) -> None:
        """Inside a streaming scope (contiguous or paged): feed each listed stream its own input frames, feeds {stream:
        int64 [K, T_s]}, through the temporal transformer only (KV and position counter advance by T_s; no text head, no
        depth steps).  The other streams are untouched.  The frames of all listed streams are packed into ragged chunks
        of at most MAX_ROWS rows (GPT.prefill_streams' row map).  On a paged scope each stream must hold pages for the
        positions it writes, or this raises before any launch."""
        self._st().prefill_streams(feeds)

    @torch.no_grad()
    @on_own_device
    def forward_depformer(self, depformer_cb_index: int, sequence: torch.Tensor, transformer_out: torch.Tensor):
        B, K, S = sequence.shape
        assert K == 1, f"Codebooks for Depformer streaming should be passed 1 by 1, got {K}."
        assert S == 1, f"Steps for Depformer streaming should be passed 1 by 1, got {S}."
        assert transformer_out.shape[1] == 1, "Transformer out should be a for a single step."
        return self._st().forward_codecformer(depformer_cb_index, sequence, transformer_out)

    @torch.no_grad()
    @on_own_device
    def forward(self, sequence: torch.Tensor, masks: Optional[torch.Tensor] = None):
        """models/model.py (MLLM_v2) :297-319, the teacher-forced forward: forward_text over [initial token,
        sequence[:, :, :-1]], then forward_local started from depformer_text_emb of each INPUT frame's text token and fed
        the input frames' audio tokens 1..dep_q.  sequence [B, K, S] -> (audio_logits [B, S, dep_q, card], text_logits
        [B, S, text_card]) in bf16, at any S (the attention window is `context` positions).  masks is accepted and unused,
        as upstream.  Evaluation only: no gradients."""
        if self._state is not None:
            raise RstnetError("LMModel.forward is the non-streaming teacher-forced form: call it outside a streaming scope")
        B, K, S = sequence.shape
        sequence = sequence.to(device=self.device, dtype=torch.int64)
        start = self._get_initial_token().repeat(B, 1, 1)
        inputs = torch.cat([start, sequence[:, :, :-1]], dim=2)
        transformer_out, text_logits = self.forward_text(inputs)
        text_logits = text_logits.squeeze(1)
        ids = inputs[:, 0, :]
        w = dict(self.named_parameters())["depformer_text_emb.weight"]
        local_start = torch.nn.functional.embedding(ids.clamp(min=0), w)
        local_start = torch.where((ids == self.zero_token_id)[..., None], torch.zeros(1, dtype=w.dtype, device=w.device), local_start)
        audio_logits = self.forward_local(local_start, inputs[:, 1:self.dep_q + 1, :], transformer_out)
        return audio_logits, text_logits


class _GenState:
    """One `LMGen.streaming(B)` scope: the delay cache with one step count per row (device), the host mirror of those
    counts, and the LMModel scope the generator drives.  The cache kernels read the LMModel scope's `active` flags."""

    def __init__(self, gen: "LMGen", lm_state: _MoshiState, B: int):
        lm = gen.lm_model
        dev, K, i64 = lm.device, lm.num_codebooks, torch.int64
        self.gen, self.lm, self.B = gen, lm_state, B
        self.cache = torch.full((B, K, gen.max_delay + 2), lm.ungenerated_token_id, device=dev, dtype=i64)
        self.off = torch.zeros(B, dtype=i64, device=dev)
        self.valid = torch.zeros(B, dtype=i64, device=dev)
        self.out = torch.zeros(B, lm.dep_q + 1, dtype=i64, device=dev)
        self.user = torch.zeros(B, K - lm.dep_q - 1, dtype=i64, device=dev)
        self.off_host = np.zeros(B, dtype=np.int64)
        self.stepped = np.zeros(B, dtype=bool)      # rows that were active in the last step

    def row_segments(self, b: int):
        """Row b's delay-cache state as row_state regions: its cache columns, step count and valid flag (`out` and `user`
        are rewritten by every step before they are read)."""
        from .row_state import tensor_segs
        return [("cache", tensor_segs(self.cache[b])), ("off", tensor_segs(self.off[b:b + 1])),
                ("valid", tensor_segs(self.valid[b:b + 1]))]

    @property
    def offset(self) -> int:
        """The reference's single step count; defined while every row is at the same step (see `off_host`)."""
        if (self.off_host != self.off_host[0]).any():
            raise RstnetError("the rows of this scope are at different steps: read off_host")
        return int(self.off_host[0])


class LMGen(nn.Module):
    """``models.model.LMGen`` (:440-597): the streaming generator over an LMModel with the acoustic-delay token cache.

    The cache keeps one step count per row, so a batch row can be restarted (`reset_streaming(streams=...)`) or held
    (`set_active_streams`) while the other rows go on; `valid_rows()` tells which rows produced output on the last step.
    A scope whose rows all start together behaves exactly as the reference."""

    def __init__(self, lm_model: LMModel, use_sampling: bool = True, temp: float = 0.8, temp_text: float = 0.7, top_k: int = 250,
                 top_k_text: int = 25, check: bool = False, top_p: float = 0.0, top_p_text: float = 0.0):
        super().__init__()
        self.lm_model = lm_model
        self.use_sampling, self.temp, self.temp_text, self.top_k, self.top_k_text, self.check = \
            use_sampling, temp, temp_text, top_k, top_k_text, check
        self.top_p, self.top_p_text = top_p, top_p_text
        if top_p or top_p_text:
            self.default_sampling()   # validates
        self._row_sampling: Optional[list] = None   # per-row Sampling once a row was given its own settings
        self.max_delay = max(lm_model.delays)
        self.delays_cuda = torch.tensor(lm_model.delays, device=lm_model.device, dtype=torch.long)
        self._st: Optional[_GenState] = None

    @property
    def is_streaming(self) -> bool:
        return self._st is not None

    def streaming_forever(self, batch_size: int, kv_pages: Optional[int] = None, kv_page: int = KV_PAGE):
        """kv_pages / kv_page: the LMModel scope's KV (LMModel.streaming_forever); a paged scope's rows hold the pages
        reserve_kv gives them."""
        lm = self.lm_model
        lm.streaming_forever(batch_size, kv_pages=kv_pages, kv_page=kv_page)
        self._st = _GenState(self, lm._st(), batch_size)
        self._row_sampling = None

    @contextmanager
    def streaming(self, batch_size: int, kv_pages: Optional[int] = None, kv_page: int = KV_PAGE):
        self.streaming_forever(batch_size, kv_pages=kv_pages, kv_page=kv_page)
        try:
            yield
        finally:
            self._st = None
            self.lm_model._state = None

    def _require(self) -> _GenState:
        if self._st is None:
            raise ValueError("the generator is not streaming")
        return self._st

    # ---- paged KV (LMGen.streaming(B, kv_pages=N)): the LMModel's methods
    def reserve_kv(self, streams, positions) -> None:
        self.lm_model.reserve_kv(streams, positions)

    def release_kv(self, streams) -> None:
        self.lm_model.release_kv(streams)

    @property
    def kv_pages_free(self) -> int:
        return self.lm_model.kv_pages_free

    @property
    def kv_page_bytes(self) -> int:
        return self.lm_model.kv_page_bytes

    def reset_streaming(self, streams=None):
        """Restart every row, or (extension) only the rows in `streams`: their cache back to ungenerated, their step count
        and their LMModel rows to 0.  The other rows and the captured graph are untouched."""
        if self._st is None:
            raise ValueError("Trying to reset streaming, but the generator wasn't streaming.")
        st = self._st
        self.lm_model.reset_streaming(streams)          # checks the row indices
        rows_h = slice(None) if streams is None else np.asarray(streams, dtype=np.int64).reshape(-1)
        rows = rows_h if streams is None else torch.from_numpy(rows_h).to(st.off.device)
        st.cache[rows] = self.lm_model.ungenerated_token_id
        st.off[rows] = 0
        st.valid[rows] = 0
        st.off_host[rows_h] = 0
        st.stepped[rows_h] = False

    def default_sampling(self) -> Sampling:
        return Sampling(bool(self.use_sampling), self.temp_text, self.top_k_text, self.top_p_text, self.temp, self.top_k, self.top_p)

    def set_stream_sampling(self, streams, sampling: Optional[Sampling] = None, seed: Optional[int] = None) -> None:
        """Extension for batched serving: give the rows in `streams` their own settings (None: the generator's) and their
        own random stream keyed by `seed` (None: 0) and the row's step count (0 at reset_streaming of the row).  From the
        first call on, every row samples through the per-row tables and keys, so a row's tokens no longer depend on which
        row it is or when it started; until then the scope draws exactly as before.  Rows reset without a seed share key 0:
        two of them with the same settings and input draw the same tokens, so pass distinct seeds to decorrelate them."""
        st = self._require()
        if sampling is not None and not isinstance(sampling, Sampling):
            raise RstnetError(f"sampling must be a Sampling (got {type(sampling).__name__})")
        rows = [int(r) for r in np.asarray(streams, dtype=np.int64).reshape(-1)]
        if any(not 0 <= r < st.B for r in rows):
            raise RstnetError(f"stream index outside [0, {st.B})")
        if self._row_sampling is None or len(self._row_sampling) != st.B:
            self._row_sampling = [self.default_sampling()] * st.B
            st.lm.row_key.zero_()
        key = int(seed or 0) & 0xFFFFFFFF
        for r in rows:
            self._row_sampling[r] = sampling if sampling is not None else self.default_sampling()
        st.lm.row_key[rows] = key - 2 ** 32 if key >= 2 ** 31 else key   # the uint32 bits

    def set_active_streams(self, mask) -> None:
        """Extension for batched serving: the rows whose flag is 0 are held by the following steps -- their cache, step
        count and LMModel rows keep their exact state.  None = every row steps."""
        self._require()
        self.lm_model.set_active_streams(mask)

    def valid_rows(self) -> np.ndarray:
        """Host bool [B]: the rows that produced output on the last step (stepped, and past their `max_delay` warm-up
        steps).  The other rows of that step's result carry no tokens."""
        st = self._require()
        return st.stepped & (st.off_host > self.max_delay)

    def get_streaming_state(self):
        """modules/streaming.py:128-136: the generator and its LMModel are one streaming module here; the state object is
        opaque and owned by the caller until it is set back."""
        return {"": self._st}

    def set_streaming_state(self, state):
        """modules/streaming.py:138-151: installs a scope of this generator (and its LMModel scope)."""
        state = dict(state)
        if "" not in state:
            raise RuntimeError("Expected to find a streaming state for .")
        st = state.pop("")
        if state:
            raise RuntimeError(f"Some states were not consumed: {list(state.keys())}")
        if st is not None and (not isinstance(st, _GenState) or st.gen is not self):
            raise RuntimeError("the streaming state belongs to another generator")
        self._st = st
        self.lm_model._state = None if st is None else st.lm

    def _frame(self, st: _GenState, force: bool = False):
        """(graph key, launch sequence): cache_in -> temporal step + text sampling + dep_q depth steps with sampling
        (sample_token over the whole card: LMGen uses plain `sample_token`, models/model.py:528-533, 581-586) -> cache_out.
        force: each sampler is followed by the forced ids of the scope's force_rows (_LMState._frame)."""
        lm, ms, L = self.lm_model, st.lm, _lib.lib()
        if self._row_sampling is not None:
            ms.set_row_sampling(self._row_sampling)     # row_valid stays 0: every row samples over the whole card
            key, frame = ms._frame(None, None, True, True, force=force)
        else:
            modes = (_head_mode(self.use_sampling, self.temp_text, self.top_k_text, self.top_p_text),
                     _head_mode(self.use_sampling, self.temp, self.top_k, self.top_p))
            key, frame = ms._frame(modes, (lm.card,) * ms.c.dep_q, False, True, force=force)
        K, CT = lm.num_codebooks, st.cache.shape[2]

        def step():
            _lib.check(L.rstnet_lm_delay_cache_in(st.cache.data_ptr(), st.off.data_ptr(), ms.active.data_ptr(),
                                                  self.delays_cuda.data_ptr(), st.user.data_ptr(), st.user.shape[1],
                                                  ms.seq.data_ptr(), ms.seq.shape[1], st.B, K, lm.dep_q, CT,
                                                  lm.text_initial_token_id, lm.initial_token_id, ops._stream()), "delay_cache_in")
            frame()
            _lib.check(L.rstnet_lm_delay_cache_out(st.cache.data_ptr(), st.off.data_ptr(), ms.active.data_ptr(),
                                                   self.delays_cuda.data_ptr(), ms.tokens.data_ptr(), ms.tokens.shape[1],
                                                   st.out.data_ptr(), st.out.shape[1], st.valid.data_ptr(), st.B, K, lm.dep_q,
                                                   CT, self.max_delay, ops._stream()), "delay_cache_out")
        return ("lmgen",) + key, step

    @torch.no_grad()
    def prefill_streams(self, prompts) -> None:
        """Extension: start rows from prompts {row: int64 [K, P]} in the step layout (`prompt_from_aligned`): rows 0..dep_q
        the tokens the row takes as sampled at steps 0..P-1, rows dep_q+1..K-1 the user tokens of those steps.  Afterwards
        the row is in the state P calls of `step` would leave it in had the sampler returned prompt[:dep_q + 1, t] at step
        t: the KV of its positions, its position counter, its delay-cache columns, step count and valid flag, and its
        per-row sampler step count (+P).  Nothing is reset: restart the rows first (reset_streaming(streams=...)) as for
        any admission; a row is taken from wherever it is.  A row with P = 0 is left as it is; every row not listed --
        live, held or mid-generation -- is untouched.  One rstnet_lm_delay_cache_prompt launch writes the cache and the
        temporal transformer's inputs, then ragged prefill chunks (the row map of LMModel.prefill_streams) run them.  On a paged scope
        each row must hold pages for min(P, context) more positions, or this raises before any launch."""
        todo = self._prompt_begin(prompts)
        while todo:
            todo = self._prompt_chunk(todo)

    def _prompt_begin(self, prompts) -> list:
        """prefill_streams up to the ragged prefill: checks, the delay-cache prompt launch, the host mirrors and step
        counts.  -> the prefill's work list for `_prompt_chunk` ([row, feed [P, K], positions fed]); until it is empty the
        rows must not step."""
        st = self._require()
        lm, ms = self.lm_model, st.lm
        K, dev = lm.num_codebooks, lm.device
        rows, parts = [], []
        for r, p in prompts.items():
            r = int(r)
            if not 0 <= r < st.B:
                raise RstnetError(f"stream index {r} outside [0, {st.B})")
            if not torch.is_tensor(p) or p.dim() != 2 or p.shape[0] != K or p.dtype.is_floating_point or p.dtype == torch.bool:
                raise RstnetError(f"the prompt of row {r} must be an integer tensor [{K}, P], got "
                                  f"{tuple(p.shape) if torch.is_tensor(p) else type(p).__name__}")
            if r in rows:
                raise RstnetError(f"row {r} is listed twice")
            rows.append(r)
            parts.append(p)
        lens = np.array([p.shape[1] for p in parts], dtype=np.int64)
        if ms.pages is not None:
            for r, n in zip(rows, lens):
                ms.pages.check([r], [ms.pos_host[r]], int(n))
        keep = [i for i in range(len(rows)) if lens[i] > 0]
        if not keep:
            return []
        rows, parts, lens = [rows[i] for i in keep], [parts[i] for i in keep], lens[keep]
        prompt = torch.cat([p.to(device=dev, dtype=torch.int64).t() for p in parts]).contiguous()     # [sum P, K]
        feed = torch.empty_like(prompt)
        starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
        r32, s32, l32 = (np.ascontiguousarray(a, dtype=np.int32) for a in (rows, starts, lens))
        _lib.check(_lib.lib().rstnet_lm_delay_cache_prompt(
            st.cache.data_ptr(), st.off.data_ptr(), st.valid.data_ptr(), self.delays_cuda.data_ptr(), prompt.data_ptr(), K,
            feed.data_ptr(), K, r32.ctypes.data, s32.ctypes.data, l32.ctypes.data, len(rows), st.B, K, lm.dep_q,
            st.cache.shape[2], self.max_delay, lm.text_initial_token_id, lm.initial_token_id, ops._stream()), "delay_cache_prompt")
        ms._cow(rows, ms.pos_host[rows], lens)
        st.off_host[rows] += lens
        idx = torch.tensor(rows, dtype=torch.int64, device=dev)
        ms.row_step.index_add_(0, idx, torch.from_numpy(lens).to(dev))
        return [[r, feed[int(a):int(a) + int(n)], 0] for r, a, n in zip(rows, starts, lens)]

    def _prompt_chunk(self, todo) -> list:
        """One ragged prefill chunk (at most MAX_ROWS rows, entries in order) of `_prompt_begin`'s work lists (several
        may be concatenated).  -> the entries not yet complete."""
        self._require().lm.row_chunk(todo)
        return [it for it in todo if it[2] < it[1].shape[0]]

    @torch.no_grad()
    def step(self, input_tokens: torch.Tensor, force: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
        """One step of every active row: -> [B, dep_q + 1, 1] in the delayed layout, or None while every row is still in
        its `max_delay` warm-up steps.  One input copy and one graph replay.

        Extension: force, an integer tensor [B, dep_q + 1, 1] (input_tokens' convention), gives the (text, audio) tokens
        the rows take at this step instead of their samples where an id is >= 0 (-1: sample), as the reference's
        depformer takes teacher-forced tokens: the forced ids feed the next depth step and the delay cache, so the next
        steps condition on them.  An id outside the head's vocabulary is not taken and sets the device error flag.  A
        graph of its own; one more copy before the replay."""
        st = self._st
        if st is None:
            raise RuntimeError("You should wrap those calls with a `with lm_gen.streaming(): ...`.")
        lm = self.lm_model
        assert input_tokens.dim() == 3, "Shape should be [B, K, T]."
        B, Ki, S = input_tokens.shape
        assert S == 1, "Only support being given steps one by one."
        needed = lm.num_codebooks - lm.dep_q - 1
        assert Ki == needed, f"We expect {needed} tokens from the user stream, got {Ki}."
        if B != st.B:
            raise RstnetError(f"streaming batch size is {st.B}, got {B}")
        ms = st.lm
        if force is not None:
            if not torch.is_tensor(force) or force.dim() != 3 or force.shape[2] != 1:
                raise RstnetError(f"force is an integer tensor [{st.B}, {lm.dep_q + 1}, 1] (-1: sample), got "
                                  f"{tuple(force.shape) if torch.is_tensor(force) else type(force).__name__}")
            ms.set_force(force[:, :, 0])
        ms._advance_host(1)
        st.user.copy_(input_tokens[:, :, 0])
        ms._replay(*self._frame(st, force is not None))
        act = ms.active_host != 0
        if self.check:
            seq = ms.seq.cpu()[torch.from_numpy(act)]
            assert not (seq == lm.ungenerated_token_id).any(), (st.off_host, seq)
        st.off_host += act
        st.stepped[:] = act
        if not (st.off_host > self.max_delay).any():
            return None
        return st.out[:, :, None].clone()


# ------------------------------------------------------------------------------------------- prompted generation
def prompt_from_aligned(seq: torch.Tensor, P: int, delays, dep_q: int, initial: int = -2) -> torch.Tensor:
    """Aligned dialogue codes seq [K, L] (rows: text, Moshi's audio codebooks 1..dep_q, then the user's audio; frame t of
    every row is time t) -> the prompt of its first P frames in LMGen's step layout, int64 [K, P], for
    LMGen.prefill_streams: forced[k, t] = seq[k, t - delays[k]] for k <= dep_q and t >= delays[k] (the token the delayed
    codebook k is sampled as at step t), `initial` where t < delays[k] (never read: LMGen feeds its initial token
    there); user[k, t] = seq[k, t] for k > dep_q (LMGen delays them itself).  P may be any length from 0 to L.

    The step layout lags codebook k by delays[k]: after the prompt, aligned frames P - max_delay .. P - 1 are only partly
    in it (codebook k holds frames < P - delays[k]).  The first max_delay steps after the prompt return aligned frames
    P - max_delay .. P - 1, whose codebooks with t + delays[k] >= P are newly sampled; steps P .. L - 1 return aligned
    frames P - max_delay .. L - 1 - max_delay."""
    if not torch.is_tensor(seq) or seq.dim() != 2 or seq.dtype.is_floating_point:
        raise RstnetError("seq must be an integer tensor [K, L]")
    K, L = seq.shape
    delays = [int(d) for d in delays]
    if len(delays) != K or min(delays) < 0:
        raise RstnetError(f"{len(delays)} delays (each >= 0) for K = {K} codebooks")
    if not 0 <= dep_q < K:
        raise RstnetError(f"dep_q = {dep_q} outside [0, {K})")
    P = int(P)
    if not 0 <= P <= L:
        raise RstnetError(f"P = {P} outside [0, {L}]")
    out = torch.empty((K, P), dtype=torch.int64, device=seq.device)
    out[:dep_q + 1] = _to_steps(seq[:dep_q + 1], delays, P, initial)
    out[dep_q + 1:] = seq[dep_q + 1:, :P]
    return out


def _to_steps(x: torch.Tensor, delays, n: int, fill: int) -> torch.Tensor:
    """Moshi's channels x [dep_q + 1, L] in the aligned layout -> their first n steps in LMGen's step layout, int64
    [dep_q + 1, n]: out[k, t] = x[k, t - delays[k]] for delays[k] <= t < L + delays[k], `fill` elsewhere (the steps that
    sample codebook k before its first aligned frame, or after the recording's last)."""
    out = torch.full((x.shape[0], n), int(fill), dtype=torch.int64, device=x.device)
    for k in range(x.shape[0]):
        d = int(delays[k])
        m = min(n - d, x.shape[1])
        if m > 0:
            out[k, d:d + m] = x[k, :m]
    return out


def force_from_aligned(seq: torch.Tensor, mask: torch.Tensor, delays, dep_q: int) -> torch.Tensor:
    """Aligned dialogue codes seq [K, L] and a bool mask [dep_q + 1, L] over Moshi's channels (text, audio codebooks
    1..dep_q; True: take seq's token at that aligned frame instead of sampling it) -> the forced ids of steps 0..L-1 in
    LMGen's step layout, int64 [dep_q + 1, L], -1 where the step samples: forced[k, t] = seq[k, t - delays[k]] where
    mask[k, t - delays[k]], the mapping prompt_from_aligned applies to the prompt.  Column t is LMGen.step's `force` at
    the row's step t; steps inside a prompt are fixed by it already."""
    if not torch.is_tensor(seq) or seq.dim() != 2 or seq.dtype.is_floating_point:
        raise RstnetError("seq must be an integer tensor [K, L]")
    K, L = seq.shape
    delays = [int(d) for d in delays]
    if len(delays) != K or min(delays) < 0:
        raise RstnetError(f"{len(delays)} delays (each >= 0) for K = {K} codebooks")
    if not 0 <= dep_q < K:
        raise RstnetError(f"dep_q = {dep_q} outside [0, {K})")
    if not torch.is_tensor(mask) or mask.dtype != torch.bool or tuple(mask.shape) != (dep_q + 1, L):
        raise RstnetError(f"a force mask is a bool tensor [{dep_q + 1}, {L}] (the item's aligned frames), got "
                          f"{(tuple(mask.shape), mask.dtype) if torch.is_tensor(mask) else type(mask).__name__}")
    vals = torch.where(mask.to(seq.device), seq[:dep_q + 1].to(torch.int64), -1)
    return _to_steps(vals, delays, L, -1)


def _item(item, K: int):
    try:
        utt, seq, P = item
    except (TypeError, ValueError):
        raise RstnetError("an item is (utt_id, seq [K, L], P)") from None
    if not torch.is_tensor(seq) or seq.dim() != 2 or seq.shape[0] != K or seq.dtype.is_floating_point:
        raise RstnetError(f"item {utt!r}: seq must be an integer tensor [{K}, L], got "
                          f"{tuple(seq.shape) if torch.is_tensor(seq) else type(seq).__name__}")
    if isinstance(P, bool) or not isinstance(P, (int, np.integer)) or not 0 <= int(P) < seq.shape[1]:
        raise RstnetError(f"item {utt!r}: P = {P!r} must be an int in [0, L = {seq.shape[1]})")
    return utt, seq, int(P)


@torch.no_grad()
def generate_many(gen: LMGen, items, capacity: int, *, seeds=None, sampling=None, kv_pages: Optional[int] = None,
                  stats: Optional[dict] = None, force=None):
    """Continuous batching of prompted Moshi generation over (utt_id, seq [K, L], P) items, seq aligned dialogue codes
    (prompt_from_aligned's layout), 0 <= P < L: yields (utt_id, out int64 [dep_q + 1, L - P]) in completion order, out
    being the aligned frames `LMGen.step` returned at steps P .. L - 1 (column j: aligned frame P + j - max_delay;
    the columns of steps below max_delay carry no frame).  An item's row is prefilled with its first P frames
    (LMGen.prefill_streams; rows admitted together share ragged chunks), then steps once per frame, fed its own
    recorded user tokens seq[dep_q + 1:, t] at step t, and finishes after step L - 1.

    Up to `capacity` items are live, one row each of an `LMGen.streaming(capacity)` scope the call opens (the generator
    must not be streaming) and closes; one graph replay per frame.  Every row samples with its own settings
    (sampling {utt_id: Sampling}; default the generator's) and random stream (seeds {utt_id: int}; default 0): an item's
    output depends on its seed and settings only, not on its row, its admission or the other items, at a given capacity.
    kv_pages N: a paged scope of N pages of KV_PAGE positions; an item holds pages for min(L, context) positions while it
    is live, and waits for them while a row is free (an item needing more than the pool raises).  Paged and contiguous
    scopes give the same tokens.  stats: a dict that receives 'frames' (steps run), 'row_frames' (live rows summed over
    steps) and 'prefill_rows' (prompt frames prefilled).

    force: {utt_id: bool mask [dep_q + 1, L]} over the item's aligned frames of Moshi's channels: where True the row
    takes seq's token at that frame instead of sampling it (force_from_aligned maps the mask to the steps; frames inside
    the prompt are fixed by it already), so every forced position of `out` equals the recording.  Forcing the audio
    codebooks and sampling the text transcribes the recording's Moshi channel; forcing the text re-voices it.  The
    per-row step tables stay on the device and are gathered by each row's step count, as the user tokens are.  Items
    without an entry run exactly as without `force` (the forced frame with nothing forced draws what the plain frame
    draws).  A mask of the wrong shape or a forced id outside its head's vocabulary raises at the item's admission."""
    lm = gen.lm_model
    K, dq = lm.num_codebooks, lm.dep_q
    Ku = K - dq - 1
    if isinstance(capacity, bool) or not isinstance(capacity, int) or not 1 <= capacity <= MAX_STREAMS:
        raise RstnetError(f"capacity must be an int in [1, {MAX_STREAMS}] (got {capacity!r})")
    if gen.is_streaming:
        raise RstnetError("generate_many opens its own streaming scope: call it on a generator that is not streaming")
    for name, d in (("seeds", seeds), ("sampling", sampling), ("force", force)):
        if d is not None and not isinstance(d, dict):
            raise RstnetError(f"{name} must be a dict keyed by utt_id")
    for s in (sampling or {}).values():
        if not isinstance(s, Sampling):
            raise RstnetError(f"sampling values must be Sampling (got {type(s).__name__})")
    seeds, sampling, force = seeds or {}, sampling or {}, force or {}
    dev = lm.device
    vocab = (lm.config.padded_vocab_size,) + (lm.card,) * dq   # the heads' vocabularies: text, then audio
    counts = dict(frames=0, row_frames=0, prefill_rows=0)
    it = iter(items)
    nxt = None
    gen.streaming_forever(capacity, kv_pages=kv_pages)
    try:
        st = gen._st
        gen.set_stream_sampling([])                 # per-row settings and random streams from the start
        pages = st.lm.pages
        free = list(range(capacity))
        live = {}                                    # row -> (utt_id, L, P, index of its first step in `hist`)
        ubuf = torch.zeros(capacity, Ku, 1, dtype=torch.int64, device=dev)   # each row's user tokens by step
        fbuf = torch.full((capacity, dq + 1, 1), -1, dtype=torch.int32, device=dev) if force else None   # ... forced ids
        hist: List[torch.Tensor] = []                # st.out after each step, from global step `base` on
        base = 0
        mask = None
        done = False
        while True:
            admitted = {}
            while free and not done:
                if nxt is None:
                    try:
                        nxt = _item(next(it), K)
                    except StopIteration:
                        done = True
                        break
                utt, seq, P = nxt
                L = seq.shape[1]
                steps = _forced_steps(utt, seq, force.get(utt), lm.delays, dq, vocab) if utt in force else None
                if pages is not None:
                    need = pages.pages_for(min(L, lm.context))
                    if need > pages.n_pages:
                        raise RstnetError(f"item {utt!r} needs {need} KV pages, the pool has {pages.n_pages}")
                    if need > pages.free:
                        break
                r = free.pop(0)
                gen.reset_streaming(streams=[r])
                gen.set_stream_sampling([r], sampling.get(utt), seeds.get(utt, 0))
                if pages is not None:
                    gen.reserve_kv([r], L)
                seq = seq.to(device=dev, dtype=torch.int64)
                if L > ubuf.shape[2]:
                    grown = torch.zeros(capacity, Ku, L, dtype=torch.int64, device=dev)
                    grown[:, :, :ubuf.shape[2]] = ubuf
                    ubuf = grown
                    if fbuf is not None:
                        grown = torch.full((capacity, dq + 1, L), -1, dtype=torch.int32, device=dev)
                        grown[:, :, :fbuf.shape[2]] = fbuf
                        fbuf = grown
                ubuf[r, :, :L] = seq[dq + 1:]
                if fbuf is not None:
                    fbuf[r] = -1
                    if steps is not None:
                        fbuf[r, :, :L] = steps.to(device=dev, dtype=torch.int32)
                admitted[r] = prompt_from_aligned(seq, P, lm.delays, dq)
                live[r] = (utt, L, P, base + len(hist))
                nxt = None
            if admitted:
                gen.prefill_streams(admitted)
                counts["prefill_rows"] += sum(p.shape[1] for p in admitted.values())
            if not live:
                if not done:
                    raise RstnetError("no item could be admitted into an empty scope")
                break
            rows = sorted(live)
            want = np.zeros(capacity, dtype=np.int64)
            want[rows] = 1
            if mask is None or not np.array_equal(mask, want):
                gen.set_active_streams(want)
                mask = want
            # each row's user tokens at its own step count (held rows read a clamped column and are not stepped)
            off = st.off.clamp(max=ubuf.shape[2] - 1)[:, None, None]
            frc = None if fbuf is None else fbuf.gather(2, off.expand(capacity, dq + 1, 1))
            gen.step(ubuf.gather(2, off.expand(capacity, Ku, 1)), force=frc)
            hist.append(st.out.clone())
            counts["frames"] += 1
            counts["row_frames"] += len(rows)
            for r in rows:
                utt, L, P, first = live[r]
                if int(st.off_host[r]) == L:
                    del live[r]
                    if pages is not None:
                        gen.release_kv([r])
                    free.append(r)
                    free.sort()
                    out = torch.stack(hist[first - base:], 2)[r]        # [dep_q + 1, L - P]
                    yield utt, out.cpu()
            first = min((v[3] for v in live.values()), default=base + len(hist))
            del hist[:first - base]
            base = first
    finally:
        gen._st = None
        lm._state = None
        if stats is not None:
            stats.update(counts)


def _forced_steps(utt, seq: torch.Tensor, mask, delays, dep_q: int, vocab) -> torch.Tensor:
    """generate_many's admission check and step table of one forced item: force_from_aligned, with every forced id
    inside its head's vocabulary"""
    try:
        steps = force_from_aligned(seq, mask, delays, dep_q)
    except RstnetError as e:
        raise RstnetError(f"item {utt!r}: {e}") from None
    for k, V in enumerate(vocab):
        row = seq[k][mask[k].to(seq.device)]
        if row.numel() and (int(row.min()) < 0 or int(row.max()) >= V):
            raise RstnetError(f"item {utt!r}: a forced id of channel {k} lies outside [0, {V})")
    return steps


# ------------------------------------------------------------------------------------------- teacher-forced scoring
AUDIO_WEIGHTS = (100, 1, 1, 1, 1, 1, 1, 1)   # validate_model's audio loss weights (MLLM/trainer/finetuning_full_fsdp.py:274-297)


def _score_metrics(sums_audio: torch.Tensor, sums_text: torch.Tensor, frames: int, audio_weights) -> dict:
    a, t = combine_sums(sums_audio, audio_weights), combine_sums(sums_text, [1])
    return {"frames": frames, "loss_audio": float(a["loss"]), "loss_text": float(t["loss"]),
            "acc_audio": float(a["acc_all"]), "acc_text": float(t["acc_all"]),
            "acc_target_audio": float(a["acc_target"]), "acc_target_text": float(t["acc_target"]),
            "sums_audio": sums_audio.tolist(), "sums_text": sums_text.tolist()}


@torch.no_grad()
def score_many(lm: LMModel, items, capacity: int = 8, audio_weights=AUDIO_WEIGHTS, ignore_audio: int = 2048,
               ignore_text: int = 32000):
    """validate_model (MLLM/trainer/finetuning_full_fsdp.py:274-297) over a corpus of (utt_id, seq [K, L], mask [K, L])
    items, K = n_q + 1: yields (utt_id, metrics) in completion order, each utterance scored as
    CrossEntropyAndAccuracy(LMModel.forward(seq)) on it alone.  metrics: loss_audio (sum_k w_k * loss_k over the dep_q
    audio codebooks with audio_weights, NOT divided by dep_q), loss_text, acc_audio / acc_text (acc_all), acc_target_audio /
    acc_target_text, frames scored, and the per-codebook sums sums_audio [dep_q][5], sums_text [1][5] (lm.CE_FIELDS).
    Trailing all-zero-mask frames are dropped; there is no length limit.  A codebook whose mask is zero throughout gives
    NaN, as upstream.  The depth transformer reads each row's own input frame (MLLM_v2's forward).

    Up to `capacity` utterances are live, one stream each of a scratch scope whose rings hold context + MAX_ROWS - 1
    positions (about 1.64 GB per stream at 7B shapes, freed when scoring ends); their frames are packed into ragged chunks
    of at most MAX_ROWS rows (lm.score_packed)."""
    if len(audio_weights) != lm.dep_q:
        raise RstnetError(f"{len(audio_weights)} audio loss weights for dep_q = {lm.dep_q} codebooks")
    if not 1 <= capacity <= MAX_STREAMS:
        raise RstnetError(f"capacity must be in [1, {MAX_STREAMS}] (got {capacity})")
    lm._check_runnable()
    K = lm.num_codebooks
    st = lm._scratch_state(capacity)
    for utt, sa, stx, L in score_packed(lm, st, items, capacity, ignore_text, ignore_audio, "inputs",
                                        lambda seq, mask: score_item(seq, mask, K)):
        yield utt, _score_metrics(sa, stx, L, audio_weights)
