"""Batched real-time frame scheduler: the serving loop of MLLM_v2/moshi/server.py:44-166 (one websocket session,
batch 1: `mimi.encode(chunk)` -> `lm_gen.step(codes)` -> `mimi.decode(tokens)` per 80 ms of audio, :108-144) generalised to
a BATCH of sessions that share one streaming scope on one GPU (SURVEY.md §8f-1, BASELINE cfg 5).

What the batch form needs beyond the reference's all-or-nothing streaming state, and where it lives:
  * admission of a new session into a free batch row of a LIVE scope   -> `reset_streaming(streams=[row])`
  * a row that delivered no audio this tick must keep its exact state  -> `set_active_streams(mask)` (the carry copy and
    the position counters of held rows do not advance; codec.py / lm.py)
  * no re-capture of CUDA graphs when sessions come and go            -> all of the above are device-side flags/counters
The websocket / Opus transport of server.py (:98-103, 141-153, 163) is out of scope (SURVEY.md §8: networking); sessions
push raw PCM chunks of 80 ms and receive (tokens, PCM) per tick.  The codec runs at 24 kHz; a `DuplexEngine` built with
another client `sample_rate` resamples every row on the GPU on the way in and on the way out (rstnet_b200.audio), so its
sessions push and receive PCM at their own rate.

`FrameScheduler` is pure host logic over an engine object with `reset_rows(rows)` and `step(pcm_rows, active) ->
{row: (tokens, pcm)}`; `DuplexEngine` is that engine for a MimiCodec + GPT pair on a GPU, `MoshiDuplexEngine` for the
MimiCodec + `LMGen(LMModel)` pair server.py itself runs (rstnet_b200.moshi).

Paged KV (`kv_pages=N` on either engine): the LM scope keeps its KV in a shared pool of N pages, and a session holds pages
only for the frames it has run -- one at admission, one more each time it crosses a page boundary, all returned when it
ends.  The engine then also has `grow_kv(rows)`, `release_rows(rows)` and `kv_pages_free` (`_PagedRows`), and the
scheduler admits on free pages and evicts a session whose next page the pool cannot give.
"""
from __future__ import annotations

import math
import time
from collections import deque
from typing import Deque, Dict, Hashable, List, Optional, Tuple

import numpy as np
import torch

from ._lib import RstnetError
from .audio import StreamingResampler
from .lm import KV_PAGE, MAX_STREAMS, Sampling

FRAME_SAMPLES = 1920       # 80 ms at 24 kHz = one 12.5 Hz frame (moshi/server.py:57: sample_rate / frame_rate)
FRAME_SECONDS = 0.08
CODEC_RATE = 24000


def check_client_rate(sample_rate) -> int:
    """A client rate r works iff gcd(r, 24000) is a multiple of 25: then 80 ms (2r/25 samples) is a whole number of
    resampling blocks in both directions (r -> 24 kHz and 24 kHz -> r).  Covers 8, 11.025, 16, 22.05, 32, 44.1 and 48 kHz."""
    if isinstance(sample_rate, bool) or not isinstance(sample_rate, (int, float)) or int(sample_rate) != sample_rate \
            or int(sample_rate) <= 0 or math.gcd(int(sample_rate), CODEC_RATE) % 25 != 0:
        raise RstnetError(f"unsupported client sample rate {sample_rate!r}: a rate r must be a positive integer with "
                          f"gcd(r, {CODEC_RATE}) % 25 == 0 (so that 80 ms is a whole number of resampling blocks)")
    return int(sample_rate)


class FrameScheduler:
    """Rows of a fixed-capacity batch are leased to sessions.  Every `tick()` steps the engine once for all rows that
    have a full frame of audio queued; the others are held.

    On an engine with paged KV (its `kv_pages` is not None) a session also holds KV pages: admission takes its first page
    and refuses while fewer than 1 + kv_headroom pages are free (kv_headroom: pages left for the live sessions to grow
    into); every tick first grows the ready sessions oldest first, and one whose next page the pool cannot give is
    evicted -- its row and pages returned, its queued frames dropped, not stepped -- and reported by `take_evicted()`."""

    def __init__(self, engine, capacity: int, kv_headroom: int = 0):
        self.engine, self.capacity = engine, capacity
        self.paged = getattr(engine, "kv_pages", None) is not None
        if isinstance(kv_headroom, bool) or not isinstance(kv_headroom, int) or kv_headroom < 0:
            raise RstnetError(f"kv_headroom must be an int >= 0 (got {kv_headroom!r})")
        self.kv_headroom = kv_headroom
        self._row_of: Dict[Hashable, int] = {}     # in admission order
        self._free: List[int] = list(range(capacity))
        self._queue: Dict[Hashable, Deque] = {}
        self._evicted: List[Hashable] = []
        self.ticks = 0

    # ---- session lifecycle
    def admit(self, session: Hashable, sampling=None, seed: Optional[int] = None) -> int:
        """Lease the lowest free row to `session` and restart that row's streaming state (server.py:156-158 does
        `mimi.reset_streaming(); lm_gen.reset_streaming()` for its single session).  sampling (an lm.Sampling) / seed:
        the session's own settings and random stream, passed to the engine's reset_rows; None: the engine's defaults.
        Once any session brought settings, a session's random stream is its seed alone (None: 0): pass distinct seeds to
        keep sessions with the same settings and input apart."""
        if session in self._row_of:
            raise RuntimeError(f"session {session!r} is already admitted")
        if not self._free:
            raise RuntimeError("no free row: the batch is full")
        if self.paged and self.engine.kv_pages_free < 1 + self.kv_headroom:
            raise RuntimeError(f"the KV pool is short: {self.engine.kv_pages_free} pages free, admission needs "
                               f"1 + {self.kv_headroom} (kv_headroom)")
        self._free.sort()
        row = self._free.pop(0)
        self._row_of[session] = row
        self._queue[session] = deque()
        if sampling is None and seed is None:
            self.engine.reset_rows([row])
        else:
            self.engine.reset_rows([row], sampling=sampling, seed=seed)
        return row

    def release(self, session: Hashable) -> None:
        row = self._row_of.pop(session)
        self._queue.pop(session, None)
        self._free.append(row)
        if self.paged:
            self.engine.release_rows([row])

    def take_evicted(self) -> List[Hashable]:
        """The sessions evicted since the last call (paged KV: the pool had no page for their next frame), oldest first."""
        out, self._evicted = self._evicted, []
        return out

    def sessions(self) -> Dict[Hashable, int]:
        return dict(self._row_of)

    def free_rows(self) -> int:
        return len(self._free)

    # ---- data path
    def push(self, session: Hashable, frame) -> None:
        """Queue one 80 ms frame (1920 samples) of the session's input audio."""
        self._queue[session].append(frame)

    def tick(self) -> Dict[Hashable, Tuple]:
        """One scheduler period: step every session that has a frame queued; returns {session: (tokens, pcm)}."""
        ready = {s: r for s, r in self._row_of.items() if self._queue[s]}
        self.ticks += 1
        if self.paged and ready:
            short = set(self.engine.grow_kv(list(ready.values())))     # admission order: the oldest sessions grow first
            for s in [s for s, r in ready.items() if r in short]:
                del ready[s]
                self.release(s)
                self._evicted.append(s)
        if not ready:
            return {}
        pcm_rows = {r: self._queue[s].popleft() for s, r in ready.items()}
        out = self.engine.step(pcm_rows, sorted(pcm_rows))
        return {s: out[r] for s, r in ready.items()}


class _PagedRows:
    """The paged-KV policy of both duplex engines, over the LM whose scope holds the pages (`_kv_lm`: a GPT, or the
    LMGen's LMModel; None: contiguous rings).  Positions come from the scope's host mirror, so no call here waits on
    the GPU, and every table change is uploaded outside graph replay (PagedKVModel.reserve_kv)."""

    kv_pages: Optional[int] = None
    _kv_lm = None

    def _reserve_first_page(self, rows) -> None:
        """A restarted row returns its old pages and holds its first page (its other pages go back to the pool)."""
        if self._kv_lm is not None:
            self._kv_lm.reserve_kv(list(rows), self._kv_lm._paged().pages.page)

    def grow_kv(self, rows) -> List[int]:
        """Walk `rows` in order: a row whose next position lies past its pages gets one more page while the pool has
        one.  A row that holds its whole ring needs none.  -> the rows that could not get their page (unchanged)."""
        st = self._kv_lm._paged()
        kp = st.pages
        grow, want, short = [], [], []
        free = kp.free
        for r in rows:
            r = int(r)
            if st.pos_host[r] + 1 <= kp.limit[r]:
                continue
            positions = (int(kp.held[r]) + 1) * kp.page
            extra = kp.pages_for(positions) - int(kp.held[r])    # 0: the last page of the ring is already held
            if extra > free:
                short.append(r)
                continue
            free -= extra
            grow.append(r)
            want.append(positions)
        if grow:
            self._kv_lm.reserve_kv(grow, want)      # one reservation and one table upload, pages handed out in row order
        return short

    def release_rows(self, rows) -> None:
        """Return the rows' pages to the pool (the rows stay in the batch, held until they are restarted)."""
        self._kv_lm.release_kv(list(rows))

    @property
    def kv_pages_free(self) -> int:
        return self._kv_lm.kv_pages_free


class DuplexEngine(_PagedRows):
    """One streaming scope of a MimiCodec and a GPT for `capacity` sessions: per tick, for all rows at once,
    encode the sessions' 80 ms chunks -> one LM frame (temporal step + 8 depth steps + sampling) -> decode the generated
    codes (the three calls of server.py:128-136).  The LM input frame of a row is [its previous text token, the 8 codes of
    its input audio]; the generated audio codes are restricted to ids < 2048 (decodable).

    `sample_rate` is the sessions' PCM rate (see `check_client_rate`): each pushes and receives sample_rate * 0.08 samples
    per tick.  At any rate other than 24000 two StreamingResamplers run for all rows at once, r -> 24 kHz before the
    encode and 24 kHz -> r after the decode; row resets and the held-row mask apply to both.

    kv_pages N: the GPT scope keeps its KV in a pool of N pages of kv_page positions (see `_PagedRows`); a restarted row
    holds one page.  None: contiguous rings."""

    def __init__(self, codec, gpt, capacity: int, *, use_sampling: bool = True, temp_text: float = 0.7, top_k_text: int = 25,
                 temp: float = 0.8, top_k: int = 30, sample_rate: int = CODEC_RATE, top_p_text: float = 0.0, top_p: float = 0.0,
                 kv_pages: Optional[int] = None, kv_page: int = KV_PAGE):
        self.sample_rate = check_client_rate(sample_rate)
        self.frame_samples = self.sample_rate * 2 // 25                       # 80 ms at the client rate
        if capacity > MAX_STREAMS:
            raise RstnetError(f"the LM step takes at most {MAX_STREAMS} streams per scope (one weight-streaming GEMM pass), "
                              f"got {capacity}")
        self.codec, self.gpt, self.B = codec, gpt, capacity
        self.dev = gpt.device
        self.sampling = dict(use_sampling=use_sampling, temp_text=temp_text, top_k_text=top_k_text, temp=temp, top_k=top_k)
        if top_p_text or top_p:
            self.sampling.update(top_p_text=top_p_text, top_p=top_p)
        self._defaults = (use_sampling, temp_text, top_k_text, top_p_text, temp, top_k, top_p)
        self.row_sampling: Optional[List[Sampling]] = None   # per-row settings once a session brought its own
        self.row_keys = np.zeros(capacity, dtype=np.int64)
        self._keys_dirty = False
        self._valid_table = None
        codec.streaming_forever(capacity)
        if kv_pages is None:
            gpt.streaming_forever(capacity)
        else:
            gpt.streaming_forever(capacity, kv_pages=kv_pages, kv_page=kv_page)
            self.kv_pages, self._kv_lm = kv_pages, gpt
        F = self.frame_samples
        self.pcm_in = torch.zeros(capacity, 1, F, dtype=torch.float32).pin_memory()
        self.pcm_dev = torch.zeros(capacity, 1, FRAME_SAMPLES, dtype=torch.float32, device=self.dev)
        self.up = self.down = None
        if self.sample_rate != CODEC_RATE:
            self.up = StreamingResampler(self.sample_rate, CODEC_RATE, capacity, self.dev)
            self.down = StreamingResampler(CODEC_RATE, self.sample_rate, capacity, self.dev)
            self.pcm_client_dev = torch.zeros(capacity, 1, F, dtype=torch.float32, device=self.dev)
            self.pcm_out_dev = torch.zeros(capacity, F, dtype=torch.float32, device=self.dev)
        self.prev_text = torch.full((capacity, 1, 1), gpt.text_initial_token_id, dtype=torch.int64, device=self.dev)
        self.tok_host = torch.zeros(capacity, gpt.config.dep_q + 1, dtype=torch.int64).pin_memory()
        self.pcm_host = torch.zeros(capacity, 1, F, dtype=torch.float32).pin_memory()
        self.mask_host = torch.zeros(capacity, dtype=torch.int64).pin_memory()
        self.latencies_ms: List[float] = []

    def reset_rows(self, rows, sampling=None, seed: Optional[int] = None) -> None:
        """Restart `rows`.  sampling / seed give them their own settings and random stream (keyed by the seed and the
        row's own frame count); from the first such call on, every row samples through per-row tables and keys, so a
        session's tokens do not depend on its row or its admission tick.  Until then the engine draws exactly as before.
        A session's random stream is its seed alone (None: 0): two sessions with the same settings, seed and input draw the
        same tokens, so callers that want them decorrelated pass distinct seeds."""
        if sampling is not None and not isinstance(sampling, Sampling):
            raise RstnetError(f"sampling must be a Sampling (got {type(sampling).__name__})")
        if sampling is not None or seed is not None or self.row_sampling is not None:
            default = Sampling(*self._defaults)
            if self.row_sampling is None:
                self.row_sampling = [default] * self.B
            for r in rows:
                self.row_sampling[r] = sampling if sampling is not None else default
                self.row_keys[r] = int(seed or 0) & 0xFFFFFFFF
            self._keys_dirty = True
        self._reserve_first_page(rows)
        self.codec.reset_streaming(streams=list(rows))
        self.gpt.reset_streaming(streams=list(rows))
        self.prev_text[list(rows)] = self.gpt.text_initial_token_id
        if self.up is not None:
            self.up.reset(rows)
            self.down.reset(rows)

    @torch.no_grad()
    def step(self, pcm_rows: Dict[int, torch.Tensor], active: List[int]):
        t0 = time.perf_counter()
        self.mask_host.zero_()
        for r, chunk in pcm_rows.items():
            self.pcm_in[r, 0].copy_(torch.as_tensor(chunk, dtype=torch.float32).reshape(self.frame_samples))
            self.mask_host[r] = 1
        self.codec.set_active_streams(self.mask_host)
        self.gpt.set_active_streams(self.mask_host)
        if self.up is None:
            self.pcm_dev.copy_(self.pcm_in, non_blocking=True)
        else:
            self.up.set_active(self.mask_host)
            self.down.set_active(self.mask_host)
            self.pcm_client_dev.copy_(self.pcm_in, non_blocking=True)
            self.up(self.pcm_client_dev[:, 0], out=self.pcm_dev[:, 0])                  # r -> 24 kHz, all rows
        codes = self.codec.encode(self.pcm_dev)                                   # [B, 8, 1]
        frame = torch.cat([self.prev_text, codes], dim=1)                        # [B, 9, 1]
        if self.row_sampling is None:
            toks = self.gpt.forward_step(frame, audio_valid=2048, **self.sampling)    # [B, 9]
        else:
            if self._valid_table is None:
                self._valid_table = torch.full((self.B, self.gpt.config.dep_q), 2048, dtype=torch.int32, device=self.dev)
            toks = self.gpt.forward_step(frame, audio_valid=self._valid_table, sampling=self.row_sampling,
                                         sample_key=self.row_keys if self._keys_dirty else None)
            self._keys_dirty = False
        held = (self.mask_host == 0).to(self.dev)
        self.prev_text.copy_(torch.where(held[:, None, None], self.prev_text, toks[:, :1, None]))
        pcm = self.codec.decode(toks[:, 1:, None].clamp(max=self.codec.codebook_size - 1))   # [B, 1, 1920]
        if self.down is not None:
            pcm = self.down(pcm[:, 0], out=self.pcm_out_dev)[:, None]                  # 24 kHz -> r, all rows
        self.tok_host.copy_(toks, non_blocking=True)
        self.pcm_host.copy_(pcm, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.latencies_ms.append(1e3 * (time.perf_counter() - t0))
        return {r: (self.tok_host[r].clone(), self.pcm_host[r, 0].clone()) for r in active}


class MoshiDuplexEngine(_PagedRows):
    """The serving loop of server.py:128-136 -- `mimi.encode -> lm_gen.step(codes) -> mimi.decode(tokens[:, 1:])` --
    for `capacity` sessions in one streaming scope of a MimiCodec and an `LMGen` (rstnet_b200.moshi).

    Every session has its own warm-up: `LMGen` returns no tokens for a row's first `max_delay` steps, and for those steps
    the codec's decoder is held for that row (the reference does not call `mimi.decode` then) while its encoder advances.
    `step` returns {row: (tokens, pcm)}, tokens = int64 [dep_q + 1] (text token, then the audio codes that were decoded),
    pcm = float32 [sample_rate * 0.08]; a row in its warm-up gets (None, None), as the reference's `lm_gen.step` returns
    None.  Text-piece decoding and the transport stay with the caller.  `sample_rate` and `kv_pages` / `kv_page` as for
    `DuplexEngine` (the pages are the LMGen's LMModel scope's)."""

    def __init__(self, codec, lm_gen, capacity: int, *, sample_rate: int = CODEC_RATE, kv_pages: Optional[int] = None,
                 kv_page: int = KV_PAGE):
        self.sample_rate = check_client_rate(sample_rate)
        self.frame_samples = self.sample_rate * 2 // 25                       # 80 ms at the client rate
        if capacity > MAX_STREAMS:
            raise RstnetError(f"the LM step takes at most {MAX_STREAMS} streams per scope (one weight-streaming GEMM pass), "
                              f"got {capacity}")
        lm = lm_gen.lm_model
        n_user = lm.num_codebooks - lm.dep_q - 1
        if codec.n_q != n_user:
            raise RstnetError(f"the codec emits {codec.n_q} codes per frame, the LM takes {n_user} user codebooks")
        self.codec, self.lm_gen, self.B = codec, lm_gen, capacity
        self.dev = lm.device
        codec.streaming_forever(capacity)
        if kv_pages is None:
            lm_gen.streaming_forever(capacity)
        else:
            lm_gen.streaming_forever(capacity, kv_pages=kv_pages, kv_page=kv_page)
            self.kv_pages, self._kv_lm = kv_pages, lm
        F = self.frame_samples
        pin = self.dev.type == "cuda"                                           # False: host logic under a test's fakes
        self.pcm_in = torch.zeros(capacity, 1, F, dtype=torch.float32, pin_memory=pin)
        self.pcm_dev = torch.zeros(capacity, 1, FRAME_SAMPLES, dtype=torch.float32, device=self.dev)
        self.up = self.down = None
        if self.sample_rate != CODEC_RATE:
            self.up = StreamingResampler(self.sample_rate, CODEC_RATE, capacity, self.dev)
            self.down = StreamingResampler(CODEC_RATE, self.sample_rate, capacity, self.dev)
            self.pcm_client_dev = torch.zeros(capacity, 1, F, dtype=torch.float32, device=self.dev)
            self.pcm_out_dev = torch.zeros(capacity, F, dtype=torch.float32, device=self.dev)
        self.tok_host = torch.zeros(capacity, lm.dep_q + 1, dtype=torch.int64, pin_memory=pin)
        self.pcm_host = torch.zeros(capacity, 1, F, dtype=torch.float32, pin_memory=pin)
        self.mask_host = torch.zeros(capacity, dtype=torch.int64, pin_memory=pin)
        self.dec_mask_host = torch.zeros(capacity, dtype=torch.int64, pin_memory=pin)
        self.dec_mask_dev = torch.zeros(capacity, dtype=torch.int64, device=self.dev)
        self.latencies_ms: List[float] = []

    def reset_rows(self, rows, sampling=None, seed: Optional[int] = None) -> None:
        """Restart `rows`; sampling / seed as DuplexEngine.reset_rows (LMGen.set_stream_sampling)."""
        self._reserve_first_page(rows)
        self.codec.reset_streaming(streams=list(rows))
        self.lm_gen.reset_streaming(streams=list(rows))
        if sampling is not None or seed is not None or getattr(self.lm_gen, "_row_sampling", None) is not None:
            self.lm_gen.set_stream_sampling(list(rows), sampling, seed)
        if self.up is not None:
            self.up.reset(rows)
            self.down.reset(rows)

    @torch.no_grad()
    def step(self, pcm_rows: Dict[int, torch.Tensor], active: List[int]):
        t0 = time.perf_counter()
        self.mask_host.zero_()
        for r, chunk in pcm_rows.items():
            self.pcm_in[r, 0].copy_(torch.as_tensor(chunk, dtype=torch.float32).reshape(self.frame_samples))
            self.mask_host[r] = 1
        self.codec.set_active_streams(self.mask_host)
        self.lm_gen.set_active_streams(self.mask_host)
        if self.up is None:
            self.pcm_dev.copy_(self.pcm_in, non_blocking=True)
        else:
            self.up.set_active(self.mask_host)
            self.pcm_client_dev.copy_(self.pcm_in, non_blocking=True)
            self.up(self.pcm_client_dev[:, 0], out=self.pcm_dev[:, 0])                  # r -> 24 kHz, all rows
        codes = self.codec.encode(self.pcm_dev)                                   # [B, 8, 1]
        toks = self.lm_gen.step(codes)                                           # [B, dep_q + 1, 1] or None
        valid = self.lm_gen.valid_rows()                                         # host mirror: no device sync
        if toks is not None:
            # rows in their warm-up keep their decoder state: decode mask = active & valid, a device-to-device copy
            self.dec_mask_host.copy_(torch.from_numpy(valid.astype("int64")))
            self.dec_mask_dev.copy_(self.dec_mask_host, non_blocking=True)
            self.codec.set_active_streams(self.dec_mask_dev)
            pcm = self.codec.decode(toks[:, 1:].clamp(0, self.codec.codebook_size - 1))   # [B, 1, 1920]
            if self.down is not None:
                self.down.set_active(self.dec_mask_dev)
                pcm = self.down(pcm[:, 0], out=self.pcm_out_dev)[:, None]                  # 24 kHz -> r, all rows
            self.tok_host.copy_(toks[:, :, 0], non_blocking=True)
            self.pcm_host.copy_(pcm, non_blocking=True)
        if self.dev.type == "cuda":
            torch.cuda.current_stream(self.dev).synchronize()
        self.latencies_ms.append(1e3 * (time.perf_counter() - t0))
        return {r: (self.tok_host[r].clone(), self.pcm_host[r, 0].clone()) if valid[r] else (None, None) for r in active}
