"""H100-native Mimi codec behind the reference's Python API.

Mirrors (names, signatures, tensor layouts, state_dict keys):
  * ``MimiCodec.encode(audio[B,1,L]) -> codes[B,n_q,ceil(L/1920)] int64`` and
    ``MimiCodec.decode(codes[B,n_q,T]) -> wav[B,1,1920*T]``
    (MLLM_v2/tools/tokenizer/MimiCodec/model/models/MimiCodec.py:25-110);
  * the ``StreamingModule`` protocol used by ``MimiModel`` under ``with m.streaming(B):`` /
    ``streaming_forever`` / ``reset_streaming`` (MLLM_v2/modules/streaming.py:33-151,
    MLLM_v2/moshi/models/compression.py:368-423): chunked encode/decode with conv carry rows and
    ring KV caches kept in device buffers;
  * ``MimiTokenizer.tokenize / detokenize`` (tools/tokenizer/MimiCodec/mimi_tokenizer.py:56-82).

All arithmetic runs in librstnet_b200.so (hand-written sm_90a CUDA); this file only lays out
buffers in HBM and sequences launches.  Internal activation layout is [B, T, C] (channels last)
so that every conv is a GEMM over overlapping contiguous rows; each layer's input buffer carries
its own left context rows (`k - stride`), which double as the streaming carry.
"""
from __future__ import annotations

import math
from contextlib import contextmanager
from typing import Dict, Iterable, Iterator, List, Optional, Tuple

import numpy as np
import torch
from torch import nn

from . import ops
from ._lib import ACT_ELU, ACT_GELU, ACT_NONE, RstnetError
from .row_state import segs, tensor_segs


def on_own_device(fn):
    """Run an API method with the module's CUDA device current: the C ABI launches on the calling thread's current
    device, while the reference lets a model live on any device regardless of it."""
    import functools

    @functools.wraps(fn)
    def wrapper(self, *a, **kw):
        dev = self.device
        if dev.type != "cuda" or torch.cuda.current_device() == (dev.index if dev.index is not None else torch.cuda.current_device()):
            return fn(self, *a, **kw)
        with torch.cuda.device(dev):
            return fn(self, *a, **kw)
    return wrapper


class _Node(nn.Module):
    """Anonymous container so that parameters get the reference's dotted state_dict names."""


def _register(root: nn.Module, dotted: str, tensor: torch.Tensor, buffer: bool = False) -> None:
    *path, leaf = dotted.split(".")
    m = root
    for p in path:
        if p not in m._modules:
            m.add_module(p, _Node())
        m = m._modules[p]
    if buffer:
        m.register_buffer(leaf, tensor)
    else:
        m.register_parameter(leaf, nn.Parameter(tensor, requires_grad=False))


_OLD_CODEBOOK_NAMES = {"inited": "_initialized", "cluster_size": "cluster_usage", "embed_avg": "embedding_sum",
                       "embed_sum": "embedding_sum"}  # quantization/core_vq.py:126-140


class MimiCodec(nn.Module):
    """Drop-in for the reference ``MimiCodec`` (same constructor arguments and defaults)."""

    def __init__(self, sample_rate=24000, n_filters=64, encoder_rates=[4, 5, 6, 8], compress=2, causal=True,
                 latent_dim=512, codebook_size=4096, codebook_dim=32, rvq_layers=8, num_heads=8, num_layers=8,
                 layer_scale=0.01, context=250, dim_feedforward=2048, semantic_feature_dim=1024,
                 target_frame_rate=12.5):
        super().__init__()
        if not causal:
            raise NotImplementedError("only the causal codec (the streaming hot path) is implemented")
        self.sample_rate = sample_rate
        self.n_filters = n_filters
        self.ratios = list(encoder_rates)
        self.compress = compress
        self.latent_dim = latent_dim
        self.codebook_size, self.codebook_dim, self.n_q, self.n_q_semantic = codebook_size, codebook_dim, rvq_layers, 1
        self.num_heads, self.num_layers = num_heads, num_layers
        self.context, self.dim_feedforward = context, 2048  # the reference hard-codes 2048 (MimiCodec.py:55)
        self.max_period = 10000.0
        self.kernel_size, self.last_kernel_size, self.residual_kernel_size = 7, 3, 3
        self.hop_length = int(math.prod(self.ratios))
        self.encoder_frame_rate = sample_rate / self.hop_length
        self.target_frame_rate = target_frame_rate
        self.resample_stride = int(self.encoder_frame_rate / self.target_frame_rate)
        self.frame_size = self.hop_length * self.resample_stride
        self.codebook_eps = 1e-5
        assert latent_dim % num_heads == 0 and n_filters % (4 * compress) == 0 and codebook_dim % 16 == 0

        D, nf = latent_dim, n_filters
        g = torch.Generator().manual_seed(0)

        def w_(shape):
            t = torch.empty(shape)
            if len(shape) >= 2:
                nn.init.xavier_uniform_(t, generator=g)
            else:
                t.zero_()
            return t

        def conv(prefix, cout, cin, k, bias=True):
            _register(self, f"{prefix}.weight", w_((cout, cin, k)))
            if bias:
                _register(self, f"{prefix}.bias", w_((cout,)))

        def resblock(prefix, dim):
            conv(f"{prefix}.block.1.conv.conv", dim // compress, dim, self.residual_kernel_size)
            conv(f"{prefix}.block.3.conv.conv", dim, dim // compress, 1)

        # encoder (modules/seanet.py:177-237)
        idx, mult = 0, 1
        conv(f"encoder.model.{idx}.conv.conv", nf, 1, self.kernel_size)
        idx += 1
        for r in reversed(self.ratios):
            resblock(f"encoder.model.{idx}", mult * nf)
            idx += 2
            conv(f"encoder.model.{idx}.conv.conv", mult * nf * 2, mult * nf, 2 * r)
            idx += 1
            mult *= 2
        idx += 1
        conv(f"encoder.model.{idx}.conv.conv", D, mult * nf, self.last_kernel_size)
        # decoder (modules/seanet.py:327-390)
        idx, mult = 0, 2 ** len(self.ratios)
        conv(f"decoder.model.{idx}.conv.conv", mult * nf, D, self.kernel_size)
        idx += 1
        for r in self.ratios:
            idx += 1
            _register(self, f"decoder.model.{idx}.convtr.convtr.weight", w_((mult * nf, mult * nf // 2, 2 * r)))
            _register(self, f"decoder.model.{idx}.convtr.convtr.bias", w_((mult * nf // 2,)))
            idx += 1
            resblock(f"decoder.model.{idx}", mult * nf // 2)
            idx += 1
            mult //= 2
        idx += 1
        conv(f"decoder.model.{idx}.conv.conv", 1, nf, self.last_kernel_size)
        s = self.resample_stride
        _register(self, "downsample.conv.conv.conv.weight", w_((D, D, 2 * s)))
        _register(self, "upsample.convtr.convtr.convtr.weight", w_((D, 1, 2 * s)))
        _register(self, "semantic_mapping_layer.ln_layer.weight", w_((D, semantic_feature_dim)))
        _register(self, "semantic_mapping_layer.ln_layer.bias", w_((D,)))
        for side in ("encoder_transformer", "decoder_transformer"):
            for l in range(num_layers):
                p = f"{side}.transformer.layers.{l}"
                _register(self, f"{p}.self_attn.in_proj_weight", w_((3 * D, D)))
                _register(self, f"{p}.self_attn.out_proj.weight", w_((D, D)))
                for n in ("norm1", "norm2"):
                    _register(self, f"{p}.{n}.weight", torch.ones(D))
                    _register(self, f"{p}.{n}.bias", torch.zeros(D))
                _register(self, f"{p}.linear1.weight", w_((self.dim_feedforward, D)))
                _register(self, f"{p}.linear2.weight", w_((D, self.dim_feedforward)))
                _register(self, f"{p}.layer_scale_1.scale", torch.full((D,), float(layer_scale)))
                _register(self, f"{p}.layer_scale_2.scale", torch.full((D,), float(layer_scale)))
        for part, n in (("rvq_first", self.n_q_semantic), ("rvq_rest", self.n_q - self.n_q_semantic)):
            _register(self, f"quantizer.{part}.input_proj.weight", w_((codebook_dim, D, 1)))
            _register(self, f"quantizer.{part}.output_proj.weight", w_((D, codebook_dim, 1)))
            for i in range(n):
                p = f"quantizer.{part}.vq.layers.{i}._codebook"
                _register(self, f"{p}._initialized", torch.tensor([False], dtype=torch.float), buffer=True)
                _register(self, f"{p}.cluster_usage", torch.ones(codebook_size), buffer=True)
                _register(self, f"{p}.embedding_sum", torch.zeros(codebook_size, codebook_dim), buffer=True)
        self._engine: Optional["_Engine"] = None
        self._stream_state: Optional["_StreamState"] = None
        self.use_cuda_graphs = True
        # streaming steps run their GEMMs on the tensor cores (wgmma, 3xTF32 = fp32-equivalent products,
        # fp32 accumulation); False selects the fp32 FFMA kernels (bit-faithful fp32 arithmetic) there too.
        self.streaming_tensor_cores = True
        # 0 = 3xTF32 (fp32-equivalent; the default on both sides: RVQ indices must match the fp32 reference and the
        # waveform stays within fp32 rounding of it).  decoder_precision = 1 opts the decoder into single-pass TF32 (the
        # precision of PyTorch's own cuDNN convolutions on GPUs): fewer MMAs, waveform error of order 1e-3 of the peak.
        self.tc_precision = 0
        self.decoder_precision = 0
        # resblock convs (k=3 C->C/2, 1x1 C/2->C) on the tensor cores too; False keeps them on the CUDA-core kernel
        self.resblock_tensor_cores = True
        # non-streaming encode / decode of a batch (offline tokenization, SURVEY.md §8f-3): batches of at least this many
        # clips run the tensor-core path (a 128-row tile = 128 clips at one time step), smaller ones the fp32 CUDA-core path
        self.batch_tensor_cores_min = 96
        self.fused_rope_attention = True     # streaming steps: RoPE + KV append inside the attention launch
        # tensor-core plans at precision 0: each 64- and 128-channel resblock is one launch (rstnet_tc_resblock) that reads
        # the raw input once and keeps the hidden tensor on chip, instead of an ELU'd copy + k3 conv + 1x1 conv
        self.fused_resblock = True
        # resblocks up to this width read the raw tensor and apply ELU in the operand transform (_Plan.elu_in_transform).
        # 0 = never (default): the ELU'd copy was the faster form where both were timed (scripts/codec_ab.py)
        self.elu_in_transform_max_channels = 0

    # ------------------------------------------------------------------ parameters
    def load_state_dict(self, state_dict, strict: bool = True, **kw):
        sd = {}
        for k, v in state_dict.items():
            head, _, leaf = k.rpartition(".")
            if head.endswith("_codebook") and leaf in _OLD_CODEBOOK_NAMES:
                k = f"{head}.{_OLD_CODEBOOK_NAMES[leaf]}"
            sd[k] = v
        self._engine = None
        return super().load_state_dict(sd, strict=strict, **kw)

    def _apply(self, fn, *a, **kw):
        self._engine = None
        return super()._apply(fn, *a, **kw)

    @classmethod
    def from_config(cls, config_path):
        import json
        with open(config_path, "r") as f:
            return cls(**json.load(f))

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    def _eng(self) -> "_Engine":
        dev = self.device
        if dev.type != "cuda":
            raise RstnetError("MimiCodec runs on CUDA only (sm_90a kernels; the CPU path is the reference itself)")
        if self._engine is None or self._engine.device != dev:
            self._engine = _Engine(self, dev)
        return self._engine

    # ------------------------------------------------------------------ reference API
    @torch.no_grad()
    @on_own_device
    def encode(self, audio_data: torch.Tensor) -> torch.Tensor:
        """[B,1,L] float -> codes [B,n_q,T] int64 (MimiCodec.py:93-101; MimiModel.encode when streaming)."""
        if audio_data.dim() != 3 or audio_data.shape[1] != 1:
            raise ValueError(f"expected audio of shape [B,1,L], got {tuple(audio_data.shape)}")
        eng = self._eng()
        x = audio_data.to(device=eng.device, dtype=torch.float32)
        if self._stream_state is not None:
            return self._stream_state.encode(x)
        return eng.encode_batch(x)

    @torch.no_grad()
    @on_own_device
    def decode(self, codes: torch.Tensor) -> torch.Tensor:
        """codes [B,K,T] int -> wav [B,1,T*frame_size] float32 (MimiCodec.py:103-110)."""
        if codes.dim() != 3:
            raise ValueError(f"expected codes of shape [B,K,T], got {tuple(codes.shape)}")
        if codes.dtype.is_floating_point:
            raise ValueError("codes must be integers")  # core_vq.py:202-204
        eng = self._eng()
        c = codes.to(device=eng.device, dtype=torch.int64).contiguous()
        if self._stream_state is not None:
            return self._stream_state.decode(c)
        return eng.decode_batch(c)

    # ------------------------------------------------------------------ corpora (continuous batching)
    def encode_many(self, items: Iterable[Tuple[object, torch.Tensor]], capacity: int = 128) -> Iterator[Tuple[object, torch.Tensor]]:
        """Encode a corpus of clips of any lengths as one continuous batch.  items: (key, wav [L] float, 24 kHz).  Yields
        (key, int64 codes [n_q, ceil(L / 1920)], on the host) as each clip finishes, equal to `encode` of that clip alone
        (bit for bit on the fp32 CUDA-core path; on the tensor cores, wherever the top-1/top-2 margin exceeds fp32 rounding).

        Up to `capacity` clips run as the rows of one streaming scope, a fixed chunk per step (CORPUS_CHUNK_FRAMES frames);
        a row whose clip ends takes the next one (per-row reset), and the chunk in which a clip ends gets the non-streaming
        right padding of the encoder's strided convs on the device (rstnet_rows_fill_tail_f32).  Independent of any
        `streaming()` scope of this codec."""
        return _corpus_run(self._eng(), items, int(capacity), "enc", CORPUS_CHUNK_FRAMES)

    def decode_many(self, items: Iterable[Tuple[object, torch.Tensor]], capacity: int = 128) -> Iterator[Tuple[object, torch.Tensor]]:
        """Decode a corpus of code sequences of any lengths as one continuous batch.  items: (key, codes [n_q, T] int).
        Yields (key, wav [1920 * T] float32, on the host) as each finishes, equal to `decode` of those codes alone.  The
        decoder is causal with no right padding, so a clip's last chunk is padded with code 0 and the output cut."""
        return _corpus_run(self._eng(), items, int(capacity), "dec", CORPUS_CHUNK_FRAMES)

    def forward(self, *a, **kw):
        raise NotImplementedError("training forward (with semantic distillation) is out of scope; use encode/decode")

    # ------------------------------------------------------------------ StreamingModule protocol
    @property
    def is_streaming(self) -> bool:
        return self._stream_state is not None

    @on_own_device
    def streaming_forever(self, batch_size: int, clip_window: bool = False):
        """clip_window (extension): the decoder transformer's rings get one step's tokens more than `context`, so every
        query sees `context` keys as in `decode` of the whole clip, and a stream of steps decodes to exactly that clip's
        `decode` at any length; False keeps the reference's RingKVCache, which leaves context - 1 keys once it wraps."""
        self._stream_state = _StreamState(self._eng(), batch_size, clip_window)

    @contextmanager
    def streaming(self, batch_size: int, clip_window: bool = False):
        self.streaming_forever(batch_size, clip_window)
        try:
            yield
        finally:
            self._stream_state = None

    @on_own_device
    def reset_streaming(self, streams=None):
        """StreamingModule.reset_streaming (modules/streaming.py:115-126).  `streams` (an extension: the reference resets
        all or nothing) restarts only those batch rows -- conv carries zeroed, transformer position counters back to 0 --
        so a frame scheduler can admit a new stream into a free row of a live batch; the other rows, the buffers and the
        captured CUDA graphs are untouched."""
        if self._stream_state is None:
            raise ValueError("Trying to reset streaming, but the codec wasn't streaming.")
        self._stream_state.reset(streams)

    def set_active_streams(self, mask) -> None:
        """Extension for batched serving (SURVEY.md §8f-1): hold the streaming state of the rows whose flag is 0 during
        the following encode / decode steps (a session that delivered no audio this tick keeps its exact state)."""
        if self._stream_state is None:
            raise ValueError("the codec is not streaming")
        self._stream_state.set_active(mask)

    def get_streaming_state(self):
        """StreamingModule.get_streaming_state (modules/streaming.py:128-136): name -> state object.  The whole codec
        is one streaming module here, so the dict has the single root entry; the object (conv carries, KV rings,
        position counters, bound launch plans) is opaque and owned by the caller until it is set back."""
        return {"": self._stream_state}

    def set_streaming_state(self, state):
        """StreamingModule.set_streaming_state (modules/streaming.py:138-151)."""
        state = dict(state)
        if "" not in state:
            raise RuntimeError("Expected to find a streaming state for .")
        st = state.pop("")
        if state:
            raise RuntimeError(f"Some states were not consumed: {list(state.keys())}")
        if st is not None and (not isinstance(st, _StreamState) or st.eng is not self._eng()):
            raise RuntimeError("the streaming state belongs to another codec (or to weights that were since reloaded / moved)")
        self._stream_state = st


class MimiTokenizer:
    """tokenize / detokenize wrapper (tools/tokenizer/MimiCodec/mimi_tokenizer.py:14-82).  The
    checkpoint download is left to the caller: pass a MimiCodec with weights loaded."""

    def __init__(self, model: MimiCodec, device=torch.device("cuda")):
        self.model = model.to(device).eval()
        self.device = device
        self.sr = 24000

    def find_length(self, x):
        return x.shape[1]

    def tokenize(self, wav, sample_rate: int = 24000):
        if not isinstance(wav, torch.Tensor):
            raise NotImplementedError
        if wav.dim() == 1:
            return wav
        if wav.dim() == 2:
            if wav.numel() == 0:
                return None
            if sample_rate != self.sr:
                raise NotImplementedError("resample to 24 kHz before tokenizing")
            wav = wav.unsqueeze(1)
        codes = self.model.encode(wav.to(self.device))
        return codes.squeeze(0).detach().cpu().to(torch.int16)

    def detokenize(self, codes):
        assert codes.shape[0] == 8
        wav = self.model.decode(codes.unsqueeze(0).to(self.device).long())
        return wav.squeeze(1).detach().cpu()


class MimiCodecBTK(MimiCodec):
    """The AudioCodec-tree variant's token layout (AudioCodec/MimiCodec/models/MimiCodec.py:94-111 with
    quantization/vq_dc.py:143-162): `encode` returns codes `[B, T, K]`, `decode` takes `[B, T, K]`.  A thin host-side
    adapter over the same kernels; that variant's third-party quantizer itself is out of scope (SURVEY.md §8c:
    `vector_quantize_pytorch` is not vendored, so the arithmetic follows the in-tree Kyutai RVQ)."""

    def encode(self, audio_data: torch.Tensor) -> torch.Tensor:
        return super().encode(audio_data).transpose(1, 2).contiguous()

    def decode(self, codes: torch.Tensor) -> torch.Tensor:
        if codes.dim() != 3:
            raise RstnetError(f"codes must be [B, T, K], got {tuple(codes.shape)}")
        return super().decode(codes.transpose(1, 2).contiguous())


# ====================================================================== engine
class _Buf:
    """fp32 activation buffer with `ctx` left-context rows: rows [ctx, ctx+T) are live, [0, ctx) is
    the causal padding / streaming carry, trailing `extra` rows are right padding.
    Layout "btc": [B, rows, C] (batch-major; FFMA path).  Layout "tbc": [rows, B, C] (time-major,
    batch-inner; a 128-row tensor-core tile = 128 streams at one time step)."""

    def __init__(self, B: int, ctx: int, T: int, extra: int, C: int, device, tbc: bool):
        self.B, self.ctx, self.T, self.extra, self.C, self.tbc = B, ctx, T, extra, C, tbc
        self.rows = ctx + T + extra
        if tbc:
            self.t = torch.zeros(self.rows, B, C, device=device, dtype=torch.float32)
            self.ts, self.bs = B * C, C
        else:
            self.t = torch.zeros(B, self.rows, C, device=device, dtype=torch.float32)
            self.ts, self.bs = C, self.rows * C

    def off(self, row: int) -> int:
        return row * self.ts

    def zero_ctx(self, streams=None):
        if self.ctx:
            if streams is None:
                (self.t[:self.ctx] if self.tbc else self.t[:, :self.ctx]).zero_()
            elif self.tbc:
                self.t[:self.ctx, streams] = 0.0
            else:
                self.t[streams, :self.ctx] = 0.0

    def row_segments(self, b: int) -> np.ndarray:
        """The carry rows [0, ctx) of stream b as state segments (row_state): ctx rows of C floats, row after row, in
        either layout."""
        if not self.ctx:
            return segs()
        e = self.t.element_size()
        if self.tbc:
            return segs((self.t.data_ptr() + b * self.bs * e, self.ts * e, self.C * e, self.ctx))
        n = self.ctx * self.C * e
        return segs((self.t.data_ptr() + b * self.bs * e, n, n, 1))

    def carry_entry(self):
        """row-copy table entry that moves the last ctx rows to the front (streaming carry)."""
        if self.tbc:
            return (self.t, 0, self.B * self.C, self.T, 0, self.ctx, self.C)
        return (self.t, self.bs, self.C, self.T, 0, self.ctx, self.C)


class _Engine:
    """Device-resident packed weights + launch sequences."""

    BATCH_MODE_BYTES = 12 << 30  # activation budget per non-streaming pass; larger batches are split

    def __init__(self, m: "MimiCodec", device: torch.device):
        self.m, self.device = m, device
        sd = {k: v.detach().to(device=device, dtype=torch.float32) for k, v in m.state_dict().items()}
        self.D, self.nf = m.latent_dim, m.n_filters
        self.ratios = list(m.ratios)
        self.enc_ratios = list(reversed(m.ratios))
        D = self.D

        def conv_w(prefix):
            """[Cout,Cin,k] -> Wt[(tap,ci), co] for the FFMA kernel and W[co, (tap,ci)] for the tensor-core GEMM."""
            w = sd[f"{prefix}.weight"]
            cout, cin, k = w.shape
            wk = w.permute(0, 2, 1).reshape(cout, k * cin).contiguous()
            return dict(W=wk, Wt=wk.t().contiguous(), bias=sd.get(f"{prefix}.bias"), taps=k)

        def convtr_w(prefix, s):
            """[Cin,Cout,2s] -> 2-tap GEMM weights: K = (half, ci) with half 0 multiplying x[t-1]
            (kernel tap j+s) and half 1 multiplying x[t] (tap j); N = (j, co)."""
            w = sd[f"{prefix}.weight"]
            cin, cout, k = w.shape
            assert k == 2 * s
            w_prev = w[:, :, s:].permute(2, 1, 0).reshape(s * cout, cin)
            w_cur = w[:, :, :s].permute(2, 1, 0).reshape(s * cout, cin)
            wk = torch.cat([w_prev, w_cur], 1).contiguous()
            return dict(W=wk, Wt=wk.t().contiguous(), bias=sd[f"{prefix}.bias"].repeat(s).contiguous(), taps=2)

        def lin_w(w):
            w = w.contiguous()
            return dict(W=w, Wt=w.t().contiguous(), bias=None, taps=1)

        # ---- encoder
        self.e_conv0_w = sd["encoder.model.0.conv.conv.weight"].reshape(self.nf, -1).contiguous()
        self.e_conv0_b = sd["encoder.model.0.conv.conv.bias"]
        self.e_res, self.e_down = [], []
        idx = 1
        for r in self.enc_ratios:
            self.e_res.append((conv_w(f"encoder.model.{idx}.block.1.conv.conv"), conv_w(f"encoder.model.{idx}.block.3.conv.conv")))
            idx += 2
            self.e_down.append(conv_w(f"encoder.model.{idx}.conv.conv"))
            idx += 1
        idx += 1
        self.e_final = conv_w(f"encoder.model.{idx}.conv.conv")
        self.down_w = conv_w("downsample.conv.conv.conv")
        # ---- decoder
        self.d_conv0 = conv_w("decoder.model.0.conv.conv")
        self.d_tr, self.d_res = [], []
        idx = 1
        for r in self.ratios:
            idx += 1
            self.d_tr.append(convtr_w(f"decoder.model.{idx}.convtr.convtr", r))
            idx += 1
            self.d_res.append((conv_w(f"decoder.model.{idx}.block.1.conv.conv"), conv_w(f"decoder.model.{idx}.block.3.conv.conv")))
            idx += 1
        idx += 1
        wf = sd[f"decoder.model.{idx}.conv.conv.weight"]  # [1, nf, k]
        self.d_final_w = wf[0].t().contiguous().reshape(-1)  # (tap, ci)
        self.d_final_b = sd[f"decoder.model.{idx}.conv.conv.bias"]
        self.up_w = sd["upsample.convtr.convtr.convtr.weight"].reshape(D, -1).contiguous()
        # ---- transformers
        self.tr = {}
        for side in ("encoder_transformer", "decoder_transformer"):
            layers = []
            for l in range(m.num_layers):
                p = f"{side}.transformer.layers.{l}"
                layers.append(dict(
                    in_w=lin_w(sd[f"{p}.self_attn.in_proj_weight"]), out_w=lin_w(sd[f"{p}.self_attn.out_proj.weight"]),
                    n1w=sd[f"{p}.norm1.weight"], n1b=sd[f"{p}.norm1.bias"],
                    n2w=sd[f"{p}.norm2.weight"], n2b=sd[f"{p}.norm2.bias"],
                    w1=lin_w(sd[f"{p}.linear1.weight"]), w2=lin_w(sd[f"{p}.linear2.weight"]),
                    ls1=sd[f"{p}.layer_scale_1.scale"], ls2=sd[f"{p}.layer_scale_2.scale"]))
            self.tr[side] = layers
        hd = D // m.num_heads
        # freqs exactly as rope.py:36-37 evaluates them (fp32 tensor * python scalar, then exp)
        ds = torch.arange(hd // 2, dtype=torch.float32)
        self.freqs = torch.exp(ds * (-math.log(m.max_period) * 2 / hd)).to(device)
        # ---- quantizer: both input projections as one GEMM (N = 2*cd), both output projections as one (K = 2*cd)
        cd = m.codebook_dim
        w1 = sd["quantizer.rvq_first.input_proj.weight"].reshape(cd, D)
        w2 = sd["quantizer.rvq_rest.input_proj.weight"].reshape(cd, D)
        self.q_in = lin_w(torch.cat([w1, w2], 0))                              # [2cd, D]
        o1 = sd["quantizer.rvq_first.output_proj.weight"].reshape(D, cd)
        o2 = sd["quantizer.rvq_rest.output_proj.weight"].reshape(D, cd)
        self.q_out = lin_w(torch.cat([o1, o2], 1))                             # [D, 2cd]
        prefixes = [f"quantizer.rvq_first.vq.layers.{i}._codebook" for i in range(m.n_q_semantic)]
        prefixes += [f"quantizer.rvq_rest.vq.layers.{i}._codebook" for i in range(m.n_q - m.n_q_semantic)]
        # centroids = embedding_sum / cluster_usage.clamp(min=eps) (core_vq.py:142-150); the squared
        # norms are taken on the host with the same ATen ops the reference's cdist uses
        embs = [sd[f"{p}.embedding_sum"].cpu() / sd[f"{p}.cluster_usage"].cpu().clamp(min=m.codebook_eps)[:, None] for p in prefixes]
        E = torch.stack(embs)
        self.E = E.contiguous().to(device)
        self.Et = E.transpose(1, 2).contiguous().to(device)
        self.enorm = E.pow(2).sum(dim=-1).contiguous().to(device)
        self.zero_counter = torch.zeros(1, dtype=torch.int64, device=device)
        self._plans: Dict[tuple, object] = {}

    # ------------------------------------------------------------------ plans
    def enc_plan(self, B: int, L: int) -> "_EncPlan":
        tc = B >= self.m.batch_tensor_cores_min
        key = ("enc", B, L, tc)
        if key not in self._plans:
            for k in [k for k in self._plans if k[0] == "enc"]:  # keep one batch-mode plan per kind alive
                del self._plans[k]
            self._plans[key] = _EncPlan(self, B, L, streaming=False, tensor_cores=tc)
        return self._plans[key]

    def dec_plan(self, B: int, T: int) -> "_DecPlan":
        tc = B >= self.m.batch_tensor_cores_min
        key = ("dec", B, T, tc)
        if key not in self._plans:
            for k in [k for k in self._plans if k[0] == "dec"]:
                del self._plans[k]
            self._plans[key] = _DecPlan(self, B, T, streaming=False, tensor_cores=tc)
        return self._plans[key]

    # ------------------------------------------------------------------ non-streaming entry points
    def encode_batch(self, x: torch.Tensor) -> torch.Tensor:
        B, _, L = x.shape
        m = self.m
        if L == 0:
            return torch.empty((B, m.n_q, 0), dtype=torch.int64, device=self.device)
        per_stream = 4 * L * (self.nf * 3.6) + (1 << 20)
        sub = max(1, min(B, int(self.BATCH_MODE_BYTES // per_stream)))
        outs = []
        for b0 in range(0, B, sub):
            xb = x[b0:b0 + sub]
            outs.append(self.enc_plan(xb.shape[0], L).run(xb, None).clone())
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    def decode_batch(self, codes: torch.Tensor) -> torch.Tensor:
        B, K, T = codes.shape
        m = self.m
        if T == 0:
            return torch.empty((B, 1, 0), dtype=torch.float32, device=self.device)
        per_stream = 4 * T * m.frame_size * (self.nf * 3.6) + (1 << 20)
        sub = max(1, min(B, int(self.BATCH_MODE_BYTES // per_stream)))
        outs = []
        for b0 in range(0, B, sub):
            cb = codes[b0:b0 + sub].contiguous()
            outs.append(self.dec_plan(cb.shape[0], T).run(cb, None).clone())
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)


def _ceil_div(a: int, b: int) -> int:
    return -(-a // b)


class _Plan:
    """Common machinery: a plan is a list of launch closures over static buffers.

    tensor_cores=False: [B, rows, C] buffers + the fp32 FFMA strided-row GEMM (exact fp32 arithmetic;
    any batch / clip length).  tensor_cores=True: [rows, B, C] buffers + wgmma 3xTF32 GEMM plans
    (streaming steps: every 128-row tile is 128 streams at one time step)."""

    def __init__(self, eng: _Engine, B: int, streaming: bool, tensor_cores: bool, active: Optional[torch.Tensor] = None,
                 corpus: bool = False):
        self.eng, self.B, self.streaming, self.tc = eng, B, streaming, tensor_cores
        self.active = active   # [B] int64 flags shared by the scope's plans: 0 = hold this stream's state this step
        self.corpus = corpus   # streaming step of the corpus drivers (encode_many / decode_many): see ring_cap
        self.ops_list = []
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.precision = eng.m.decoder_precision if isinstance(self, _DecPlan) else eng.m.tc_precision

    def buf(self, ctx, T, extra, C) -> _Buf:
        return _Buf(self.B, ctx, T, extra, C, self.eng.device, self.tc)

    def elu_in_transform(self, C: int) -> bool:
        """Tensor-core plans: does the resblock conv of a C-channel level apply its input ELU in the GEMM's operand transform
        (reading the raw tensor) instead of reading an ELU'd copy written by the producer?  Same values either way (one
        ELU implementation, bit-identical results).  The idea: at the wide, shallow levels (24 kHz C = 64, 6 kHz C = 128)
        the copy is a second 126 / 63 MB tensor per 256-stream frame.  Where it was timed (scripts/codec_ab.py) it did not
        pay -- the extra ex2 per operand element cost more than the saved stores -- so
        MimiCodec.elu_in_transform_max_channels defaults to 0; time it with scripts/codec_ab.py before changing that."""
        return self.tc and C <= self.eng.m.elu_in_transform_max_channels and self.precision == 0 and self.eng.m.resblock_tensor_cores

    def fused_resblock(self, C: int) -> bool:
        """Tensor-core plans: is the C-channel resblock one rstnet_tc_resblock launch?  It reads the raw tensor (the buffer
        layout of elu_in_transform: the raw tensor owns the carry rows, no ELU'd copy) and keeps the hidden tensor in
        shared memory.  Same values as the two-launch form, bit for bit."""
        return (self.tc and C in (64, 128) and self.precision == 0 and self.eng.m.resblock_tensor_cores
                and self.eng.m.fused_resblock)

    def raw_resblock_input(self, C: int) -> bool:
        """Does the resblock input buffer itself carry the causal context (no separate ELU'd copy)?"""
        return not self.tc or self.elu_in_transform(C) or self.fused_resblock(C)

    def resblock(self, y: _Buf, ya: _Buf, h: Optional[_Buf], w1, w2, out: _Buf, T: int):
        """SEANetResnetBlock (ELU, k3 C -> C/2, ELU, 1x1 C/2 -> C, + skip) followed by ELU: out rows [out.ctx, +T) from y
        rows [y.ctx, +T).  ya: the buffer the k3 conv reads, with the 2 causal context rows: y itself, or the ELU'd copy
        its producer wrote.  h: the hidden tensor (None when the block is fused)."""
        if self.fused_resblock(y.C):
            assert ya is y and y.ctx == 2 and self.tc
            B = self.B
            w1_hi, w1_lo = self.tc_weights(w1)
            w2_hi, w2_lo = self.tc_weights(w2)
            plan = ops.TcResblock(y.t, 0, y.C, B * y.C, y.rows, B, T, w1_hi, w1_lo, w1["bias"], w2_hi, w2_lo, w2["bias"],
                                  out.t, out.off(out.ctx), out.C, B * out.C)
            self.add(plan.run)
            return
        self.conv(ya, 0, 1, w1, h, 0, T, pre=ACT_ELU if ya is y else ACT_NONE, post=ACT_ELU, ffma=self.tc)
        self.conv(h, 0, 1, w2, out, out.ctx, T, post=ACT_ELU, R=y, r_row0=y.ctx, ffma=self.tc)

    @staticmethod
    def tc_weights(pack):
        """TF32 (hi, lo) split of a weight pack, computed once and cached on the pack."""
        if "W_hi" not in pack:
            pack["W_hi"], pack["W_lo"] = ops.tf32_split(pack["W"])
        return pack["W_hi"], pack["W_lo"]

    def add(self, fn):
        self.ops_list.append(fn)

    def launch(self):
        for fn in self.ops_list:
            fn()

    # ---- conv / transposed conv over a _Buf (taps along time)
    def conv(self, A: _Buf, a_row0: int, stride: int, pack, out: _Buf, out_row0: int, T_out: int, *, pre=ACT_NONE,
             post=ACT_NONE, R: Optional[_Buf] = None, r_row0: int = 0, tr_stride: int = 0, out2: Optional[_Buf] = None,
             out2_row0: int = 0, ffma: bool = False):
        """out2 (tensor-core plans only): ELU'd copy of the raw output, written by the same epilogue, so the
        consumer that needs a pre-activation (resblock conv1) does not re-apply ELU per tap and per N tile."""
        B, Cin = self.B, A.C
        taps = pack["taps"]
        N = pack["W"].shape[0]
        if not self.tc:
            kw = dict(bias=pack["bias"], pre_act=pre, post_act=post)
            if R is not None:
                kw.update(R=R.t, r_off=R.off(r_row0), r_bs=R.bs, r_rs=R.ts)
            self.add(lambda: ops.gemm_rows(A.t, A.off(a_row0), A.bs, stride * Cin, pack["Wt"], out.t, out.off(out_row0),
                                           out.bs, N, B, T_out, **kw))
            return
        if ffma and (Cin % 32 != 0 or self.precision != 0 or not self.eng.m.resblock_tensor_cores):
            # time-major layout on the CUDA cores: rows of a "batch" = the B streams of one output time step, taps are
            # B*Cin apart.  Fallback for the resblock convs (single-pass TF32 decoder option, or
            # resblock_tensor_cores = False to compare against the CUDA-core path).
            assert not tr_stride and out2 is None
            kw = dict(bias=pack["bias"], pre_act=pre, post_act=post, taps=taps, tap_stride=B * Cin)
            if R is not None:
                kw.update(R=R.t, r_off=R.off(r_row0), r_bs=B * R.C, r_rs=R.C)
            self.add(lambda: ops.gemm_rows(A.t, A.off(a_row0), stride * B * Cin, Cin, pack["Wt"], out.t, out.off(out_row0),
                                           B * out.C, out.C, T_out, B, **kw))
            return
        kw = dict(taps=taps, tap_do=1, o_mul=stride, bias=pack["bias"], pre_act=pre, post_act=post, precision=self.precision)
        if R is not None:
            kw.update(R=R.t, r_off=R.off(r_row0), r_i_stride=R.C, r_o_stride=B * R.C)
        if tr_stride:
            kw.update(n_split=out.C, c_split_stride=B * out.C)
        if out2 is not None:
            kw.update(C2=out2.t, c2_off=out2.off(out2_row0), act2=ACT_ELU)
        w_hi, w_lo = self.tc_weights(pack)
        plan = ops.TcGemm(A.t, A.off(a_row0), Cin, B * Cin, Cin, B, A.rows - a_row0, w_hi, Cin, out.t, out.off(out_row0),
                          out.C, (tr_stride or 1) * B * out.C, B, T_out, W_lo=w_lo, **kw)
        self.add(plan.run)

    # ---- linear over `rows` consecutive rows
    def linear(self, A_t, a_rows_view, K, pack, out_t, out_view, N_row_stride, *, post=ACT_NONE, scale=None, R_view=None):
        """a_rows_view / out_view / R_view: (offset, batch, rows_per_batch, batch_stride) with row stride K / N_row_stride."""
        a_off, nb, rpb, a_bs = a_rows_view
        c_off, _, _, c_bs = out_view
        if not self.tc:
            kw = dict(post_act=post, scale=scale)
            if R_view is not None:
                kw.update(R=out_t, r_off=R_view[0], r_bs=R_view[3], r_rs=N_row_stride)
            self.add(lambda: ops.gemm_rows(A_t, a_off, a_bs, K, pack["Wt"], out_t, c_off, c_bs, N_row_stride, nb, rpb, **kw))
            return
        assert nb == 1
        kw = dict(post_act=post, scale=scale, precision=self.precision)
        if R_view is not None:
            kw.update(R=out_t, r_off=R_view[0], r_i_stride=N_row_stride, r_o_stride=rpb * N_row_stride)
        w_hi, w_lo = self.tc_weights(pack)
        plan = ops.TcGemm(A_t, a_off, K, rpb * K, K, rpb, 1, w_hi, K, out_t, c_off, N_row_stride, rpb * N_row_stride, rpb, 1,
                          W_lo=w_lo, **kw)
        self.add(plan.run)

    def rows_view(self, X: _Buf, row0: int, nrows: int):
        """(offset, batch, rows_per_batch, batch_stride) of rows [row0, row0+nrows) of every stream."""
        if self.tc:
            return (X.off(row0), 1, nrows * self.B, 0)
        return (X.off(row0), self.B, nrows, X.bs)

    def flat_view(self, nrows: int, width: int):
        """a contiguous [B*nrows, width] scratch in the plan's row order."""
        if self.tc:
            return (0, 1, nrows * self.B, 0)
        return (0, self.B, nrows, nrows * width)

    def ring_cap(self, F: int) -> int:
        """KV slots of the transformer.  Non-streaming: the whole clip (linear buffer).  Streaming: `context`, the
        reference's RingKVCache, whose labelling leaves only cap - 1 keys attendable once it wraps (codec_attn.cu).  The
        corpus drivers promise the non-streaming result, where every query sees `context` keys, so their rings have F
        more slots than the window: the clamp end - cap + 1 then never binds."""
        if not self.streaming:
            return F
        return self.eng.m.context + (F if self.corpus else 0)

    # ---- the 8-layer codec transformer, in place on rows [x_row, x_row+F) of X
    def transformer(self, side: str, X: _Buf, x_row: int, F: int, cap: int):
        eng, m, B = self.eng, self.eng.m, self.B
        D, H, FF = eng.D, m.num_heads, m.dim_feedforward
        hd = D // H
        dev = eng.device
        ln = torch.empty(B * F, D, device=dev)
        qkv = torch.empty(B * F, 3 * D, device=dev)
        att = torch.empty(B * F, D, device=dev)
        ff = torch.empty(B * F, FF, device=dev)
        self.scratch = (ln, qkv, att, ff)
        if self.streaming:
            kv = [torch.zeros(2, B, H, cap, hd, device=dev) for _ in range(m.num_layers)]
            offset = torch.zeros(B, dtype=torch.int64, device=dev)   # one position counter per stream (per-stream reset)
        else:
            kv = [torch.zeros(2, B, H, cap, hd, device=dev)] * m.num_layers
            offset = eng.zero_counter
        self.kv, self.offset, self.cap = kv, offset, cap
        xv = self.rows_view(X, x_row, F)
        if self.tc:
            q_bs, q_ts, o_bs, o_ts = 3 * D, B * 3 * D, D, B * D
            ln_args = (1, F * B)
        else:
            q_bs, q_ts, o_bs, o_ts = F * 3 * D, 3 * D, F * D, D
            ln_args = (B, F)
        x_bs = 0 if self.tc else X.bs
        linear = not self.streaming
        for l, w in enumerate(eng.tr[side]):
            kvl = kv[l]
            self.add(lambda w=w: ops.layer_norm(X.t, xv[0], x_bs, w["n1w"], w["n1b"], ln, ln_args[0], ln_args[1], D, 1e-5))
            self.linear(ln, self.flat_view(F, D), D, w["in_w"], qkv, self.flat_view(F, 3 * D), 3 * D)
            if self.streaming and F == 2 and hd == 64 and m.fused_rope_attention and min(q_bs, q_ts, o_bs, o_ts) % 4 == 0:
                # one launch: the warp that owns (stream, head) rotates / appends its new k, v and attends
                self.add(lambda kvl=kvl: ops.rope_ring_attention(qkv, q_bs, q_ts, kvl, offset, eng.freqs, att, o_bs, o_ts, B, F, H, hd,
                                                                 cap, m.context))
            else:
                self.add(lambda kvl=kvl: ops.rope_kv_append(qkv, q_bs, q_ts, kvl, offset, eng.freqs, B, F, H, hd, cap))
                self.add(lambda kvl=kvl: ops.ring_attention(qkv, q_bs, q_ts, kvl, offset, att, o_bs, o_ts, B, F, H, hd, cap, m.context,
                                                            linear))
            self.linear(att, self.flat_view(F, D), D, w["out_w"], X.t, xv, D, scale=w["ls1"], R_view=xv)
            self.add(lambda w=w: ops.layer_norm(X.t, xv[0], x_bs, w["n2w"], w["n2b"], ln, ln_args[0], ln_args[1], D, 1e-5))
            self.linear(ln, self.flat_view(F, D), D, w["w1"], ff, self.flat_view(F, FF), FF, post=ACT_GELU)
            self.linear(ff, self.flat_view(F, FF), FF, w["w2"], X.t, xv, D, scale=w["ls2"], R_view=xv)

    def finish_streaming(self, carries: List[_Buf], F: int):
        if not self.streaming:
            return
        dev = self.eng.device
        self.carries = carries
        entries = [b.carry_entry() for b in carries if b.ctx]
        table = ops.make_copy_table(entries, dev)
        n, nb = len(entries), (1 if self.tc else self.B)
        self.copy_table = table
        self.add(lambda: ops.rows_copy_table(table, n, nb, self.active))
        self.add(lambda: ops.counter_add(self.offset, F, self.active))

    def row_segments(self, b: int):
        """Stream b's state in this streaming plan, as row_state regions: the carry rows of every buffer, every layer's
        transformer ring kv[l][:, b] (all `cap` slots: unwritten ones are masked by the position), the position counter."""
        regions = [(f"carry{i}", buf.row_segments(b)) for i, buf in enumerate(self.carries) if buf.ctx]
        for l, kv in enumerate(self.kv):
            e = kv.element_size()
            regions.append((f"ring{l}", segs((kv[0, b].data_ptr(), kv.stride(0) * e, kv[0, b].numel() * e, 2))))
        regions.append(("offset", tensor_segs(self.offset[b:b + 1])))
        return regions

    def reset(self, streams=None):
        assert self.streaming
        for b in self.carries:
            b.zero_ctx(streams)
        if streams is None:
            self.offset.zero_()
        else:
            self.offset[streams] = 0


class _EncPlan(_Plan):
    """Buffers + launch order of one encode pass (whole clip, or one streaming chunk)."""

    def __init__(self, eng: _Engine, B: int, L: int, streaming: bool, tensor_cores: bool, active: Optional[torch.Tensor] = None,
                 valid: Optional[torch.Tensor] = None):
        """valid (corpus streaming steps): device int64 [B], the samples of each stream's clip in this chunk; a stream
        whose clip ends inside the chunk gets the non-streaming right padding there (see tail_fill)."""
        super().__init__(eng, B, streaming, tensor_cores, active, corpus=valid is not None)
        m, dev = eng.m, eng.device
        self.L = L
        if streaming and L % m.frame_size != 0:
            raise RstnetError(f"streaming chunks must be multiples of {m.frame_size} samples, got {L}")
        nf, D = eng.nf, eng.D
        k0 = m.kernel_size
        T = [L]
        for r in eng.enc_ratios:
            T.append(_ceil_div(T[-1], r))
        self.F = F = T[-1]
        s = m.resample_stride
        self.T5 = T5 = _ceil_div(F, s)
        self.xin = xin = self.buf(k0 - 1, L, 0, 1)
        y, ya, h, r_ = [], [], [], []  # ya: ELU'd copies feeding the resblocks' first conv (tensor-core plans)
        C = nf
        for i, ratio in enumerate(eng.enc_ratios):
            own_copy = not self.raw_resblock_input(C)
            y.append(self.buf(0 if own_copy else m.residual_kernel_size - 1, T[i], 0, C))
            ya.append(self.buf(m.residual_kernel_size - 1, T[i], 0, C) if own_copy else y[-1])
            h.append(None if self.fused_resblock(C) else self.buf(0, T[i], 0, C // m.compress))
            r_.append(self.buf(ratio, T[i], T[i + 1] * ratio - T[i], C))
            C *= 2
        y4 = self.buf(m.last_kernel_size - 1, F, 0, C)
        X = self.buf(s, F, T5 * s - F, D)
        cd = m.codebook_dim
        self.lat = lat = torch.empty(B * T5, D, device=dev)
        xproj = torch.empty(B * T5, 2 * cd, device=dev)
        self.codes = codes = torch.zeros(B, m.n_q, T5, dtype=torch.int64, device=dev)
        work = torch.empty(ops.rvq_encode_workspace(B * T5, m.n_q, cd, m.codebook_size), dtype=torch.uint8, device=dev)
        self._keep = (xproj, work)

        # conv0: 1 -> nf, k7 (HBM-bound, CUDA cores)
        if self.tc and ya[0] is not y[0]:
            self.add(lambda: ops.conv1d_cin1(xin.t, xin.bs, xin.ts, eng.e_conv0_w, eng.e_conv0_b, y[0].t, 0, y[0].bs, y[0].ts, B, L,
                                             nf, k0, ACT_NONE, out2=ya[0].t, out2_off=ya[0].off(ya[0].ctx), act2=ACT_ELU))
        else:
            self.add(lambda: ops.conv1d_cin1(xin.t, xin.bs, xin.ts, eng.e_conv0_w, eng.e_conv0_b, y[0].t, y[0].off(y[0].ctx),
                                             y[0].bs, y[0].ts, B, L, nf, k0, ACT_NONE))
        for i, ratio in enumerate(eng.enc_ratios):
            w1, w2 = eng.e_res[i]
            # SEANetResnetBlock: ELU -> k3 -> ELU -> k1, + skip; the ELU that follows is fused as post_act
            self.resblock(y[i], ya[i], h[i], w1, w2, r_[i], T[i])
            if valid is not None:   # the downsampling conv's zero right padding at the end of a clip
                self.tail_fill(r_[i], T[i], 0, valid, math.prod(eng.enc_ratios[:i]))
            if i + 1 < len(y):
                nxt = y[i + 1]
                self.conv(r_[i], 0, ratio, eng.e_down[i], nxt, nxt.ctx, T[i + 1],
                          out2=ya[i + 1] if ya[i + 1] is not nxt else None, out2_row0=ya[i + 1].ctx)
            else:
                self.conv(r_[i], 0, ratio, eng.e_down[i], y4, y4.ctx, T[i + 1], post=ACT_ELU)
        self.conv(y4, 0, 1, eng.e_final, X, X.ctx, F)
        self.transformer("encoder_transformer", X, X.ctx, F, self.ring_cap(F))
        # ConvDownsample1d: replicate padding (left on the first call only when streaming)
        fill_bs, fill_nb, fill_C = (0, 1, B * D) if self.tc else (X.bs, B, D)
        only0 = self.offset if streaming else None
        self.add(lambda: ops.rows_fill(X.t, fill_bs, fill_nb, fill_C, 0, X.ctx, mode=1, src_row=X.ctx, only_if_zero=only0,
                                       channels_per_stream=D))
        if X.extra:
            self.add(lambda: ops.rows_fill(X.t, fill_bs, fill_nb, fill_C, X.ctx + X.T, X.extra, mode=1, src_row=X.ctx + X.T - 1))
        if valid is not None:       # ... and on the right at the end of a clip
            self.tail_fill(X, F, 1, valid, eng.m.hop_length)
        lat_buf = _LatView(lat, B, T5, D, self.tc)
        self.conv(X, 0, s, eng.down_w, lat_buf, 0, T5)
        self.linear(lat, self.flat_view(T5, D), D, eng.q_in, xproj, self.flat_view(T5, 2 * cd), 2 * cd)
        self.add(lambda: ops.rvq_encode(xproj, 2 * cd, eng.E, eng.Et, eng.enorm, codes, work, B * T5, T5, m.n_q, m.n_q_semantic,
                                        cd, m.codebook_size, time_major=self.tc))
        self.finish_streaming([xin] + ya + r_ + [y4, X], F)

    def tail_fill(self, X: _Buf, T: int, mode: int, valid: torch.Tensor, div: int):
        """rows [X.ctx + n_b, X.ctx + T) of stream b := 0 (mode 0) or its last valid row (mode 1), n_b = ceil(valid[b] / div):
        the length the non-streaming T chain gives this layer for the clip's remaining samples (the chunk starts at a
        multiple of every stride)."""
        bs, nb, C = (0, 1, self.B * X.C) if self.tc else (X.bs, self.B, X.C)
        self.add(lambda: ops.rows_fill_tail(X.t, bs, nb, C, X.ctx, T, mode, valid, div, channels_per_stream=X.C))

    def run(self, x: torch.Tensor, graphs: Optional[bool]) -> torch.Tensor:
        xin, L = self.xin, self.L
        if self.tc:
            xin.t[xin.ctx:xin.ctx + L, :, 0].copy_(x[:, 0, :].t())
        else:
            xin.t[:, xin.ctx:xin.ctx + L, 0].copy_(x[:, 0, :])
        _run_plan(self, graphs)
        return self.codes


class _LatView:
    """Adapter so a contiguous [B*T, C] tensor can be the output `_Buf` of `_Plan.conv`."""

    def __init__(self, t: torch.Tensor, B: int, T: int, C: int, tbc: bool):
        self.t, self.C, self.ctx, self.rows, self.tbc = t, C, 0, T, tbc
        self.ts, self.bs = (B * C, C) if tbc else (C, T * C)

    def off(self, row: int) -> int:
        return row * self.ts


class _DecPlan(_Plan):
    """Buffers + launch order of one decode pass."""

    def __init__(self, eng: _Engine, B: int, T: int, streaming: bool, tensor_cores: bool, n_codes: Optional[int] = None,
                 active: Optional[torch.Tensor] = None, corpus: bool = False):
        super().__init__(eng, B, streaming, tensor_cores, active, corpus)
        m, dev = eng.m, eng.device
        self.T = T
        D, nf = eng.D, eng.nf
        s = m.resample_stride
        self.F = F = T * s
        cd = m.codebook_dim
        K = n_codes or m.n_q
        self.codes_in = codes_in = torch.zeros(B, K, T, dtype=torch.int64, device=dev)
        q = torch.empty(B * T, 2 * cd, device=dev)
        qup = self.buf(1, T, 0, D)
        X = self.buf(m.kernel_size - 1, F, 0, D)
        C = nf * 2 ** len(eng.ratios)
        a = [self.buf(1, F, 0, C)]
        yd, yda, hd_ = [], [], []
        Tin = F
        for i, r in enumerate(eng.ratios):
            Tout = Tin * r
            own_copy = not self.raw_resblock_input(C // 2)
            yd.append(self.buf(0 if own_copy else m.residual_kernel_size - 1, Tout, 0, C // 2))
            yda.append(self.buf(m.residual_kernel_size - 1, Tout, 0, C // 2) if own_copy else yd[-1])
            hd_.append(None if self.fused_resblock(C // 2) else self.buf(0, Tout, 0, C // 2 // m.compress))
            last = i == len(eng.ratios) - 1
            a.append(self.buf((m.last_kernel_size - 1) if last else 1, Tout, 0, C // 2))
            C //= 2
            Tin = Tout
        self.Lout = Lout = Tin
        self.wav = wav = torch.empty(B, 1, Lout, device=dev)

        self.add(lambda: ops.rvq_decode_gather(codes_in, eng.E, q, B * T, T, K, m.n_q_semantic, cd, m.codebook_size,
                                               time_major=self.tc))
        self.linear(q, self.flat_view(T, 2 * cd), 2 * cd, eng.q_out, qup.t, self.rows_view(qup, 1, T), D)
        self.add(lambda: ops.convtr1d_depthwise(qup.t, qup.bs, qup.ts, eng.up_w, X.t, X.off(X.ctx), X.bs, X.ts, B, T, D, s))
        self.transformer("decoder_transformer", X, X.ctx, F, self.ring_cap(F))
        self.conv(X, 0, 1, eng.d_conv0, a[0], 1, F, post=ACT_ELU)
        Tin = F
        for i, r in enumerate(eng.ratios):
            # ConvTranspose1d k=2r stride r as a 2-tap GEMM over [x[t-1], x[t]]: one output row = r time steps
            self.conv(a[i], 0, 1, eng.d_tr[i], yd[i], yd[i].ctx, Tin, tr_stride=r, out2=yda[i] if yda[i] is not yd[i] else None,
                      out2_row0=yda[i].ctx)
            Tout = Tin * r
            w1, w2 = eng.d_res[i]
            self.resblock(yd[i], yda[i], hd_[i], w1, w2, a[i + 1], Tout)
            Tin = Tout
        last = a[-1]
        self.add(lambda: ops.conv1d_cout1(last.t, last.bs, last.ts, eng.d_final_w, eng.d_final_b, wav, Lout, B, Lout, last.C,
                                          m.last_kernel_size))
        self.finish_streaming([qup, X] + a + yda, F)
        # scripts/diag_rows.py (fused resblocks have no hidden buffer)
        self.debug_bufs = {"qup": [qup], "X": [X], "a": a, "yd": yd, "yda": yda, "hd": [b for b in hd_ if b is not None]}

    def run(self, codes: torch.Tensor, graphs: Optional[bool]) -> torch.Tensor:
        self.codes_in.copy_(codes)
        _run_plan(self, graphs)
        return self.wav


def _run_plan(plan, graphs: Optional[bool]) -> None:
    """Launch eagerly, or (streaming steps) replay a CUDA graph of the whole step: all buffers are
    static and the stream position lives in a device counter, so one capture serves every step."""
    if not graphs:
        plan.launch()
        return
    if plan.graph is None:
        plan.warmups = getattr(plan, "warmups", 0) + 1
        if plan.warmups <= 2:
            plan.launch()  # eager warm-up steps (also set the kernels' smem attributes)
            return
        torch.cuda.synchronize()
        plan.graph = ops.capture(plan.launch)  # capture only; nothing executes until replay
    plan.graph.replay()


class _StreamState:
    """Per-`streaming(B)` scope state: one encode plan and one decode plan per chunk size, sharing
    nothing with other scopes (mirrors `_MimiState`, compression.py:37-60)."""

    def __init__(self, eng: _Engine, batch_size: int, clip_window: bool = False):
        self.eng, self.B, self.clip_window = eng, batch_size, clip_window
        self.enc: Dict[int, _EncPlan] = {}
        self.dec: Dict[int, _DecPlan] = {}
        # per-stream "advance" flags read by the carry copy and the position counters of every step (all ones unless a
        # frame scheduler holds rows that received no input this tick, see set_active)
        self.active = torch.ones(batch_size, dtype=torch.int64, device=eng.device)

    def encode(self, x: torch.Tensor) -> torch.Tensor:
        B, _, L = x.shape
        if B != self.B:
            raise RstnetError(f"streaming batch size is {self.B}, got {B}")
        if L == 0:
            return torch.empty((B, self.eng.m.n_q, 0), dtype=torch.int64, device=self.eng.device)
        return self._enc_plan(L).run(x, self.eng.m.use_cuda_graphs).clone()

    def _enc_plan(self, L: int) -> "_EncPlan":
        if L not in self.enc:
            if self.enc:
                raise RstnetError("the chunk size must stay constant within one streaming scope")
            self.enc[L] = _EncPlan(self.eng, self.B, L, True, self.eng.m.streaming_tensor_cores, active=self.active)
        return self.enc[L]

    def _dec_plan(self, T: int, K: int) -> "_DecPlan":
        if T not in self.dec:
            if self.dec:
                raise RstnetError("the chunk size must stay constant within one streaming scope")
            self.dec[T] = _DecPlan(self.eng, self.B, T, True, self.eng.m.streaming_tensor_cores, n_codes=K, active=self.active,
                                   corpus=self.clip_window)
        return self.dec[T]

    def row_segments(self, b: int, chunk: int, frames: int, n_codes: int):
        """Stream b's state as row_state regions: the encoder plan of `chunk` samples and the decoder plan of `frames`
        frames of n_codes codes (built here if no step has built them yet, as encode / decode would)."""
        enc, dec = self._enc_plan(chunk), self._dec_plan(frames, n_codes)
        return [("enc." + n, s) for n, s in enc.row_segments(b)] + [("dec." + n, s) for n, s in dec.row_segments(b)]

    def decode(self, codes: torch.Tensor) -> torch.Tensor:
        B, K, T = codes.shape
        if B != self.B:
            raise RstnetError(f"streaming batch size is {self.B}, got {B}")
        return self._dec_plan(T, K).run(codes, self.eng.m.use_cuda_graphs).clone()

    def set_active(self, mask):
        """mask [B] (bool / int): streams with 0 are HELD by the next steps -- they still run through the kernels (the
        batch is one launch sequence) but their conv carries and transformer positions do not advance, so the step
        leaves no trace on them.  None = all streams advance."""
        if mask is None:
            self.active.fill_(1)
        else:
            self.active.copy_(torch.as_tensor(mask).to(device=self.eng.device, dtype=torch.int64).reshape(self.B))

    def reset(self, streams=None):
        if streams is not None:
            # checked before the copy to the device, so that a reset does not wait for the device
            streams = torch.as_tensor(streams, dtype=torch.int64).reshape(-1)
            if streams.numel() and (int(streams.min()) < 0 or int(streams.max()) >= self.B):
                raise RstnetError(f"stream index outside [0, {self.B})")
            streams = streams.to(self.eng.device)
        for p in list(self.enc.values()) + list(self.dec.values()):
            p.reset(streams)


# 12.5 Hz frames per step of encode_many / decode_many.  Measured with scripts/codec_corpus_bench.py on an H100 80GB HBM3
# at a 400 W power limit (1 024 clips of 1-40 s): 8 frames was the fastest of 1 / 2 / 4 / 8 at capacities 64, 128 and 256,
# for encode and for decode (fewer launches per frame; the padded last chunk of a clip costs 3.5 frames on average)
CORPUS_CHUNK_FRAMES = 8


class _CorpusScope:
    """The device side of encode_many / decode_many: one streaming plan of `B` rows with rings of context + T slots, and
    one staging buffer that a single host-to-device copy per step fills: per-row valid counts (encoder tail fill), the
    per-row `active` flags the plan holds idle rows with, the rows to reset before the step, and the chunk itself."""

    def __init__(self, eng: _Engine, B: int, kind: str, frames: int):
        m, dev = eng.m, eng.device
        self.eng, self.B, self.kind = eng, B, kind
        self.enc = kind == "enc"
        self.chunk = frames * m.frame_size if self.enc else frames      # samples or frames per step
        self.hdr = 3 * 8 * B
        pay_shape = (B, 1, self.chunk) if self.enc else (B, m.n_q, frames)
        pay_dtype = torch.float32 if self.enc else torch.int64
        nbytes = self.hdr + math.prod(pay_shape) * pay_dtype.itemsize
        self.stage = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        self.host = [torch.zeros(nbytes, dtype=torch.uint8).pin_memory() for _ in range(2)]
        valid, active, self.reset_rows = (self.stage[i * 8 * B:(i + 1) * 8 * B].view(torch.int64) for i in range(3))
        self.payload = self.stage[self.hdr:].view(pay_dtype).view(pay_shape)
        tc = m.streaming_tensor_cores
        if self.enc:
            self.plan = _EncPlan(eng, B, self.chunk, True, tc, active=active, valid=valid)
            out = self.plan.codes
        else:
            self.plan = _DecPlan(eng, B, frames, True, tc, active=active, corpus=True)
            out = self.plan.wav
        self.out = [torch.empty(out.shape, dtype=out.dtype).pin_memory() for _ in range(2)]
        self.events = [torch.cuda.Event() for _ in range(2)]

    def host_views(self, k: int):
        """numpy views of host staging buffer k: valid, active, reset rows, payload."""
        h = self.host[k].numpy()
        B = self.B
        valid, active, reset = (h[i * 8 * B:(i + 1) * 8 * B].view(np.int64) for i in range(3))
        return valid, active, reset, h[self.hdr:].view(np.float32 if self.enc else np.int64).reshape(self.payload.shape)

    def submit(self, k: int, n_reset: int):
        """One step from host staging buffer k; its output lands in self.out[k] when self.events[k] completes."""
        self.stage.copy_(self.host[k], non_blocking=True)
        if n_reset:
            self.plan.reset(self.reset_rows[:n_reset])
        out = self.plan.run(self.payload, self.eng.m.use_cuda_graphs)
        self.out[k].copy_(out, non_blocking=True)
        self.events[k].record()


class _Clip:
    __slots__ = ("key", "data", "n", "pos", "parts", "done", "total")

    def __init__(self, key, data: np.ndarray, n: int, total: int):
        self.key, self.data, self.n, self.total = key, data, n, total
        self.pos, self.done, self.parts = 0, 0, []


@torch.no_grad()
def _corpus_run(eng: _Engine, items, B: int, kind: str, frames: int):
    """Continuous batching of encode_many ("enc") / decode_many ("dec").  The schedule depends only on the clip lengths,
    so the host prepares step n + 1 while the device runs step n, and waits once per step, for the output of step n."""
    if B < 1:
        raise ValueError(f"capacity must be at least 1, got {B}")
    m = eng.m
    enc = kind == "enc"
    fs = m.frame_size
    with torch.cuda.device(eng.device):
        scope = _CorpusScope(eng, B, kind, frames)
    chunk = scope.chunk
    source = iter(items)
    ready = []   # clips with nothing to compute

    def next_clip() -> Optional[_Clip]:
        for key, x in source:
            if enc:
                w = torch.as_tensor(x).detach()
                if w.dim() != 1:
                    raise ValueError(f"encode_many: clip {key!r} must be a 1-D waveform [L], got {tuple(w.shape)}")
                w = np.ascontiguousarray(w.to("cpu", torch.float32).numpy())
                c = _Clip(key, w, w.shape[0], _ceil_div(w.shape[0], fs))
            else:
                cd = torch.as_tensor(x).detach()
                if cd.dim() != 2 or cd.shape[0] != m.n_q or cd.dtype.is_floating_point:
                    raise ValueError(f"decode_many: codes of {key!r} must be integers [{m.n_q}, T], got {cd.dtype} {tuple(cd.shape)}")
                cd = np.ascontiguousarray(cd.to("cpu", torch.int64).numpy())
                c = _Clip(key, cd, cd.shape[1], cd.shape[1] * fs)
            if c.n:
                return c
            ready.append((key, torch.empty((m.n_q, 0), dtype=torch.int64) if enc else torch.empty(0)))
        return None

    def harvest(k: int, records):
        scope.events[k].synchronize()
        out = scope.out[k].numpy()
        for b, c, ncols in records:
            c.parts.append(out[b, :, :ncols].copy() if enc else out[b, 0, :ncols].copy())
            c.done += ncols
            if c.done == c.total:
                ready.append((c.key, torch.from_numpy(np.concatenate(c.parts, -1))))

    rows: List[Optional[_Clip]] = [None] * B
    exhausted, pending, k = False, None, 0
    while True:
        valid, active, reset, pay = scope.host_views(k)
        n_reset, records = 0, []
        for b in range(B):
            c = rows[b]
            if c is not None and c.pos >= c.n:
                c = rows[b] = None
            if c is None and not exhausted:
                c = rows[b] = next_clip()
                if c is None:
                    exhausted = True
                else:
                    reset[n_reset] = b
                    n_reset += 1
            if c is None:
                valid[b], active[b] = chunk, 0      # held; a full chunk: no tail fill
                continue
            take = min(chunk, c.n - c.pos)
            if enc:
                pay[b, 0, :take] = c.data[c.pos:c.pos + take]
                pay[b, 0, take:] = 0.0
                records.append((b, c, _ceil_div(take, fs)))
            else:
                pay[b, :, :take] = c.data[:, c.pos:c.pos + take]
                pay[b, :, take:] = 0
                records.append((b, c, take * fs))
            valid[b], active[b] = take, 1
            c.pos += take
        if records:
            with torch.cuda.device(eng.device):
                scope.submit(k, n_reset)
        if pending is not None:
            harvest(*pending)
        yield from ready
        ready.clear()
        if not records:
            return
        pending, k = (k, records), k ^ 1
