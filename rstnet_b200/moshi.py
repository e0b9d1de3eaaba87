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

The kernels are the GPT path's (rstnet_b200/lm.py): weight-streaming wgmma GEMMs with fused Kyutai RMSNorm / SiLU gating
finalizes, ring decode attention, the depth transformer, device-side sampling; plus the bf16 pair-RoPE kernel.  One
`LMGen.step` is one CUDA-graph replay.
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
from .lm import GPT, SkinnyGemm, _DepthScope, _LMState  # noqa: F401


class _MoshiState(_LMState):
    """`_LMState` with the Kyutai temporal layer: in_proj (p h d) -> pair-RoPE -> ring attention -> out_proj, gating FFN."""

    def _pack_temporal(self, P):
        return {}

    def _build_temporal(self, P, G, z, parent):
        m, c, B, M = self.m, self.c, self.B, self.M
        dev = m.device
        E, V, I = c.n_embd, c.padded_vocab_size, c.intermediate_size
        nh, hs = c.n_head, c.head_size
        self.seq = z(M, c.n_q + 1, dtype=torch.int64)
        self.x, self.xn, self.q, self.att = z(M, E), z(M, E), z(M, E), z(M, E)
        self.qkv, self.hmid = z(M, 3 * E), z(M, I)
        self.out, self.logits = z(M, E), z(M, V)
        if parent is not None:
            raise RstnetError("the Moshi twin streams one position per call (LMGen.step)")
        self.offset = z(B, dtype=torch.int64)
        self.pos_host = np.zeros(B, dtype=np.int64)
        self.active = torch.ones(B, dtype=torch.int64, device=dev)
        self.active_host = np.ones(B, dtype=np.int64)
        self.kv = [z(2, B, nh, self.cap, hs) for _ in range(c.n_layer)]
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

    def _temporal(self, head: bool = True):
        c, B, M, L = self.c, self.B, self.M, _lib.lib()
        st = ops._stream()
        E = c.n_embd
        _lib.check(L.rstnet_lm_embed_sum_bf16(self.seq.data_ptr(), c.n_q + 1, self.wte.data_ptr(), self.wte.shape[0],
                                              self.table_ptrs.data_ptr(), self.tables[0].shape[0], c.n_q, E, self.x.data_ptr(), M, st),
                   "lm_embed_sum")
        _lib.check(L.rstnet_lm_rms_norm_bf16(self.x.data_ptr(), self.n1_first.data_ptr(), self.xn.data_ptr(), M, E, 1e-8, 1, st), "rms")
        for l, ly in enumerate(self.layers):
            ly["qkv"].run()
            _lib.check(L.rstnet_lm_rope_pair_kv_append_bf16(self.qkv.data_ptr(), self.offset.data_ptr(), 1, self.q.data_ptr(),
                                                            self.kv[l].data_ptr(), M, B, c.n_head, c.head_size, self.cap,
                                                            self.freqs.data_ptr(), st), "rope_pair_kv")
            _lib.check(L.rstnet_lm_ring_decode_attention_bf16(self.q.data_ptr(), self.kv[l].data_ptr(), self.offset.data_ptr(), 1,
                                                              self.att.data_ptr(), M, B, c.n_head, c.n_head, c.head_size, self.cap,
                                                              c.context, None, st), "attention")
            ly["proj"].run()
            ly["fc"].run()
            ly["down"].run()
        if head:
            self.head.run()
        ops.counter_add(self.offset, self.tn, self.active)

    def _advance_host(self, n: int):
        self.pos_host += n * self.active_host      # positions enter the RoPE as fp32 angles: no table to run out of


class LMModel(nn.Module):
    """Drop-in for ``models.model.LMModel`` on the streaming decode path (same constructor arguments / defaults)."""

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
        self._state: Optional[_MoshiState] = None
        self._packed = None
        self.use_cuda_graphs = True
        self.use_depth_frame_kernel = False

    # ---- state_dict keys identical to the reference (`depformer.` lives under a private name: `depformer` is an API object)
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
        sd = {}
        for k, v in state_dict.items():
            for src, dst in self._RENAME:
                if k.startswith(dst):
                    k = src + k[len(dst):]
            sd[k] = v
        self._packed = None
        return super().load_state_dict(sd, strict=strict, **kw)

    def _apply(self, fn, *a, **kw):
        self._packed = None
        return super()._apply(fn, *a, **kw)

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

    @property
    def zero_token_id(self) -> int:
        return -1

    @property
    def ungenerated_token_id(self) -> int:
        return -2

    @property
    def device(self):
        return next(iter(self.parameters())).device

    @property
    def num_codebooks(self) -> int:
        return self.n_q + 1

    @property
    def num_audio_codebooks(self) -> int:
        return self.n_q

    @property
    def audio_offset(self) -> int:
        return 1

    def _get_initial_token(self) -> torch.Tensor:
        tok = torch.full([1, self.num_codebooks, 1], self.initial_token_id, device=self.device, dtype=torch.long)
        tok[:, 0] = self.text_initial_token_id
        return tok

    # ---- streaming protocol
    @property
    def is_streaming(self) -> bool:
        return self._state is not None

    @on_own_device
    def streaming_forever(self, batch_size: int):
        if self.device.type != "cuda":
            raise RstnetError("LMModel decode runs on CUDA only (sm_90a kernels; the CPU path is the reference itself)")
        if next(self.parameters()).dtype != torch.bfloat16:
            raise RstnetError("LMModel decode runs in bfloat16: call .to(device, torch.bfloat16)")
        self._state = _MoshiState(self, batch_size)

    @contextmanager
    def streaming(self, batch_size: int):
        self.streaming_forever(batch_size)
        try:
            yield
        finally:
            self._state = None

    @on_own_device
    def reset_streaming(self, streams=None):
        if self._state is None:
            raise ValueError("Trying to reset streaming, but the model wasn't streaming.")
        self._state.reset(streams)

    def _st(self) -> _MoshiState:
        if self._state is None:
            raise RstnetError("only the streaming decode path is implemented: call inside `with lm.streaming(B):`")
        return self._state

    # ---- reference API
    @torch.no_grad()
    @on_own_device
    def forward_text(self, sequence: torch.Tensor):
        B, K, S = sequence.shape
        assert K == self.num_codebooks, f"Sequence shape {sequence.shape} must match the number of codebooks."
        if S != 1:
            raise RstnetError("streaming forward_text takes one frame per call")
        out, logits = self._st().forward_global(sequence)
        return out, logits[:, None]                                  # [B,1,dim], [B,1,1,text_card]

    @torch.no_grad()
    @on_own_device
    def forward_depformer(self, depformer_cb_index: int, sequence: torch.Tensor, transformer_out: torch.Tensor):
        B, K, S = sequence.shape
        assert K == 1, f"Codebooks for Depformer streaming should be passed 1 by 1, got {K}."
        assert S == 1, f"Steps for Depformer streaming should be passed 1 by 1, got {S}."
        assert transformer_out.shape[1] == 1, "Transformer out should be a for a single step."
        return self._st().forward_codecformer(depformer_cb_index, sequence, transformer_out)

    def forward(self, *a, **kw):
        raise NotImplementedError("training forward is out of scope; use LMGen.step / forward_text / forward_depformer")


class LMGen(nn.Module):
    """``models.model.LMGen`` (:440-597): the streaming generator over an LMModel with the acoustic-delay token cache."""

    def __init__(self, lm_model: LMModel, use_sampling: bool = True, temp: float = 0.8, temp_text: float = 0.7, top_k: int = 250,
                 top_k_text: int = 25, check: bool = False):
        super().__init__()
        self.lm_model = lm_model
        self.use_sampling, self.temp, self.temp_text, self.top_k, self.top_k_text, self.check = \
            use_sampling, temp, temp_text, top_k, top_k_text, check
        self.max_delay = max(lm_model.delays)
        self.delays_cuda = torch.tensor(lm_model.delays, device=lm_model.device, dtype=torch.long)
        self._st = None

    @property
    def is_streaming(self) -> bool:
        return self._st is not None

    def streaming_forever(self, batch_size: int):
        lm = self.lm_model
        lm.streaming_forever(batch_size)
        cache = torch.full((batch_size, lm.num_codebooks, self.max_delay + 2), lm.ungenerated_token_id, device=lm.device, dtype=torch.long)
        self._st = SimpleNamespace(cache=cache, initial=lm._get_initial_token(), offset=0)

    @contextmanager
    def streaming(self, batch_size: int):
        self.streaming_forever(batch_size)
        try:
            yield
        finally:
            self._st = None
            self.lm_model._state = None

    def reset_streaming(self):
        if self._st is None:
            raise ValueError("Trying to reset streaming, but the generator wasn't streaming.")
        self._st.offset = 0
        self.lm_model.reset_streaming()

    @torch.no_grad()
    def step(self, input_tokens: torch.Tensor) -> Optional[torch.Tensor]:
        st = self._st
        if st is None:
            raise RuntimeError("You should wrap those calls with a `with lm_gen.streaming(): ...`.")
        lm = self.lm_model
        assert input_tokens.dim() == 3, "Shape should be [B, K, T]."
        B, Ki, S = input_tokens.shape
        assert S == 1, "Only support being given steps one by one."
        needed = lm.num_codebooks - lm.dep_q - 1
        assert Ki == needed, f"We expect {needed} tokens from the user stream, got {Ki}."
        CT = st.cache.shape[2]
        for q_other in range(Ki):                                   # the user's stream goes into the cache at its delay
            k = lm.dep_q + 1 + q_other
            wp = (st.offset + lm.delays[k]) % CT
            st.cache[:, k, wp:wp + 1] = input_tokens[:, q_other]
        position = st.offset % CT
        for k, delay in enumerate(lm.delays):                        # delayed codebooks start from the initial token
            if st.offset <= delay:
                st.cache[:, k, position] = st.initial[:, k, 0]
        input_ = st.cache[:, :, position:position + 1]
        if self.check:
            assert not (input_ == lm.ungenerated_token_id).any(), (st.offset, input_)
        # temporal step + text sampling + dep_q depth steps with sampling: one graph replay (sample_token over the whole
        # card: LMGen uses plain `sample_token`, models/model.py:528-533, 581-586)
        toks = lm._st().forward_step(input_, self.use_sampling, self.temp_text, self.top_k_text, self.temp, self.top_k,
                                     lm.card, True)                  # [B, dep_q + 1]
        st.offset += 1
        position = st.offset % CT
        st.cache[:, 0, position] = toks[:, 0]
        st.cache[:, 1:lm.dep_q + 1, position] = toks[:, 1:]
        if st.offset <= self.max_delay:
            return None
        gen_delays = self.delays_cuda[:lm.dep_q + 1]
        index = ((st.offset - self.max_delay + gen_delays) % CT).view(1, -1, 1).expand(B, -1, 1)
        return st.cache.gather(dim=2, index=index)
