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

Suspend / resume (`suspend_rows(rows)` / `resume_rows(rows, states)` on either engine, paged or not; `_DuplexCore`): a
session's state -- codec carries and rings, resampler carries, the KV it wrote, counters, sampling settings -- is packed
into pinned host memory (row_state.SessionState), which frees its row and its pages; later it is unpacked into any free
row of a compatible engine, and the session goes on with the bytes an uninterrupted run would have produced.
`FrameScheduler(on_short="suspend")` suspends a session the pool cannot grow instead of evicting it.
"""
from __future__ import annotations

import math
import time
from collections import deque
from typing import Deque, Dict, Hashable, List, Optional, Tuple

import numpy as np
import torch

from . import row_state
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
    evicted -- its row and pages returned, its queued frames dropped, not stepped -- and reported by `take_evicted()`.

    Suspension (an engine with suspend_rows / resume_rows): `suspend(session)` packs the session's state into host
    memory and frees its row and pages; its queue stays, and `push` keeps queueing to it.  `resume(session)` unpacks it
    into the lowest free row.  With on_short="suspend" a session whose next page the pool cannot give is suspended
    instead of evicted, and every tick first resumes suspended sessions, oldest first, while a row and
    pages_for(its positions) + 1 + kv_headroom pages are free.  A resumed session still steps one frame per tick, so it
    lags by the ticks it spent suspended (its queue holds the frames pushed meanwhile); `lag` records them per session."""

    def __init__(self, engine, capacity: int, kv_headroom: int = 0, on_short: str = "evict"):
        self.engine, self.capacity = engine, capacity
        self.paged = getattr(engine, "kv_pages", None) is not None
        if isinstance(kv_headroom, bool) or not isinstance(kv_headroom, int) or kv_headroom < 0:
            raise RstnetError(f"kv_headroom must be an int >= 0 (got {kv_headroom!r})")
        if on_short not in ("evict", "suspend"):
            raise RstnetError(f"on_short must be 'evict' or 'suspend' (got {on_short!r})")
        self.kv_headroom, self.on_short = kv_headroom, on_short
        self._suspended: Dict[Hashable, object] = {}   # session -> SessionState, in suspension order
        self._suspended_at: Dict[Hashable, int] = {}
        self.lag: Dict[Hashable, int] = {}              # ticks each session has spent suspended
        self.suspensions = self.resumes = 0
        self._row_of: Dict[Hashable, int] = {}     # in admission order
        self._free: List[int] = list(range(capacity))
        self._queue: Dict[Hashable, Deque] = {}
        self._evicted: List[Hashable] = []
        self.ticks = 0

    # ---- session lifecycle
    def admit(self, session: Hashable, sampling=None, seed: Optional[int] = None, prompt=None) -> int:
        """Lease the lowest free row to `session` and restart that row's streaming state (server.py:156-158 does
        `mimi.reset_streaming(); lm_gen.reset_streaming()` for its single session).  sampling (an lm.Sampling) / seed:
        the session's own settings and random stream, passed to the engine's reset_rows; None: the engine's defaults.
        Once any session brought settings, a session's random stream is its seed alone (None: 0): pass distinct seeds to
        keep sessions with the same settings and input apart.

        prompt (a MoshiDuplexEngine only): int64 [K, P] in LMGen's step layout (moshi.prompt_from_aligned), the frames
        the session starts from (MoshiDuplexEngine.reset_rows).  Its prefill is spread over the following ticks, one
        ragged chunk of at most MAX_ROWS rows per tick (packing the pending prompts of every session admitted so), run
        before the tick's step; until it is complete the session is held and its pushed frames queue.  A paged engine
        needs kv_pages_for(P + 1) + kv_headroom free pages."""
        if session in self._row_of:
            raise RuntimeError(f"session {session!r} is already admitted")
        if not self._free:
            raise RuntimeError("no free row: the batch is full")
        P = 0
        if prompt is not None:
            if not hasattr(self.engine, "check_prompt"):
                raise RstnetError("prompts are a MoshiDuplexEngine feature: this engine starts sessions empty")
            P = self.engine.check_prompt(prompt)
        need = (self.engine.kv_pages_for(P + 1) if prompt is not None and self.paged else 1) + self.kv_headroom
        if self.paged and self.engine.kv_pages_free < need:
            raise RuntimeError(f"the KV pool is short: {self.engine.kv_pages_free} pages free, admission needs "
                               f"{need - self.kv_headroom} + {self.kv_headroom} (kv_headroom)")
        self._free.sort()
        row = self._free[0]
        if prompt is not None:
            self.engine.start_rows([row], sampling=sampling, seed=seed, prompts={row: prompt})
        elif sampling is None and seed is None:
            self.engine.reset_rows([row])
        else:
            self.engine.reset_rows([row], sampling=sampling, seed=seed)
        self._free.pop(0)
        self._row_of[session] = row
        self._queue[session] = deque()
        return row

    def release(self, session: Hashable) -> None:
        if session in self._suspended:       # its state and queue are dropped; it holds no row or pages
            del self._suspended[session], self._suspended_at[session]
            self._queue.pop(session, None)
            return
        row = self._row_of.pop(session)
        self._queue.pop(session, None)
        self._free.append(row)
        if row in self._prefilling():
            self.engine.drop_prefill([row])
        if self.paged:
            self.engine.release_rows([row])

    def take_evicted(self) -> List[Hashable]:
        """The sessions evicted since the last call (paged KV: the pool had no page for their next frame), oldest first."""
        out, self._evicted = self._evicted, []
        return out

    def suspend(self, session: Hashable):
        """Pack the session's state into host memory (engine.suspend_rows) and free its row and pages; its queue stays.
        -> its SessionState."""
        row = self._row_of[session]
        if row in self._prefilling():
            raise RuntimeError(f"session {session!r} is still prefilling its prompt")
        state = self.engine.suspend_rows([row])[0]
        del self._row_of[session]
        self._free.append(row)
        self._suspended[session], self._suspended_at[session] = state, self.ticks
        self.suspensions += 1
        return state

    def resume(self, session: Hashable) -> int:
        """Unpack a suspended session into the lowest free row (engine.resume_rows; a short pool raises and changes
        nothing).  -> the row."""
        if session not in self._suspended:
            raise RuntimeError(f"session {session!r} is not suspended")
        if not self._free:
            raise RuntimeError("no free row: the batch is full")
        self._free.sort()
        row = self._free[0]
        self.engine.resume_rows([row], [self._suspended[session]])
        self._free.pop(0)
        del self._suspended[session]
        self.lag[session] = self.lag.get(session, 0) + self.ticks - self._suspended_at.pop(session)
        self._row_of[session] = row
        self.resumes += 1
        return row

    def suspended(self) -> List[Hashable]:
        """The suspended sessions, oldest suspension first."""
        return list(self._suspended)

    def _resume_waiting(self) -> None:
        """on_short="suspend": resume suspended sessions, oldest first, while a row and their pages (+ 1 + kv_headroom)
        are free."""
        if self.paged:
            self.engine.reclaim()
        for s in list(self._suspended):
            if not self._free:
                return
            if self.paged and self.engine.kv_pages_free < (self.engine.kv_pages_for(max(self._suspended[s].positions, 1)) + 1
                                                            + self.kv_headroom):
                return
            self.resume(s)

    def sessions(self) -> Dict[Hashable, int]:
        return dict(self._row_of)

    def free_rows(self) -> int:
        return len(self._free)

    # ---- data path
    def push(self, session: Hashable, frame) -> None:
        """Queue one 80 ms frame (1920 samples) of the session's input audio."""
        self._queue[session].append(frame)

    def _prefilling(self):
        return getattr(self.engine, "prefilling", frozenset())

    def tick(self) -> Dict[Hashable, Tuple]:
        """One scheduler period: one chunk of the pending prompt prefills, if any, then step every session that has a
        frame queued and no prefill left; returns {session: (tokens, pcm)}."""
        if self.on_short == "suspend" and self._suspended:
            self._resume_waiting()
        if self._prefilling():
            self.engine.prefill_chunk()
        held = self._prefilling()
        ready = {s: r for s, r in self._row_of.items() if self._queue[s] and r not in held}
        self.ticks += 1
        if self.paged and ready:
            short = set(self.engine.grow_kv(list(ready.values())))     # admission order: the oldest sessions grow first
            for s in [s for s, r in ready.items() if r in short]:
                del ready[s]
                if self.on_short == "suspend":
                    self.suspend(s)
                else:
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
    the GPU, and every table change is uploaded outside graph replay (the model's reserve_kv)."""

    kv_pages: Optional[int] = None
    _kv_lm = None

    def _reserve_first_page(self, rows) -> None:
        """A restarted row returns its old pages and holds its first page (its other pages go back to the pool)."""
        if self._kv_lm is not None:
            self._kv_lm.reserve_kv(list(rows), self._kv_lm._paged().pages.page)

    def grow_kv(self, rows) -> List[int]:
        """Walk `rows` in order: a row whose next position lies past its pages gets one more page while the pool has
        one.  A row that holds its whole ring needs none.  -> the rows that could not get their page (unchanged)."""
        self.reclaim()
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
        """Pages no row holds, without the pages of suspended rows whose gather is still in flight."""
        return self._kv_lm.kv_pages_free

    def kv_pages_for(self, positions: int) -> int:
        return self._kv_lm._paged().pages.pages_for(positions)

    def reclaim(self) -> int:
        """Return the pages of suspended rows whose gather has completed to the pool (no wait).  -> pages returned."""
        n = 0
        for item in list(getattr(self, "_in_flight", ())):
            if item[0].query():
                self._kv_lm._paged().pages.give_back(item[1])
                self._in_flight.remove(item)
                n += len(item[1])
        return n


class _DuplexCore(_PagedRows):
    """What both duplex engines share: the client rate and its resamplers, the pinned host buffers, a tick's input half (PCM
    copy -> upsample -> encode) and output half (decode -> downsample -> D2H -> synchronise -> per-row results), row
    restarts, and suspend / resume.  An engine adds its LM part: `_reset_lm_rows`, `_lm_step`, and the row state of
    `_row_host` / `_row_regions` / `_set_row_host` / `_per_row_sampling`.

    Suspend / resume: the engine lists a row's state as row_state regions (`_row_regions`) and host fields (`_row_host` /
    `_set_row_host`); this class moves them with one segment gather / scatter launch per row on a side stream of at most
    `swap_ctas` CTAs.

    Ordering, with no host synchronise on the tick path:
      * suspend: the gather waits (an event) for the ticks already enqueued; the row then stays held -- a held row's
        state does not advance -- and its pages are unmapped but stay out of the pool until the gather's completion
        event has passed (`reclaim`, or the next tick).
      * resume: the scatter waits for the ticks already enqueued, for the state's gather and for any swap still touching
        the row; the next tick makes the main stream wait for the scatter (every tick runs every row of the batch, held
        ones included, so no tick may touch the row before its state has landed).
      * reset_rows of a row makes the main stream wait for every gather or scatter still touching it, so a session
        admitted into a row whose previous session was just suspended (or resumed and released) starts clean.
    Host memory: the pinned blob and table of every swap are kept by the engine until the swap has completed, so a
    caller may drop a SessionState at any time.  The blob of a resumed state returns to the engine's pool once its
    scatter has completed (the state is then consumed), and later suspends reuse pooled blobs (best fit) before they
    allocate; `pin_host_blobs` fills the pool up front so that suspension allocates nothing on the tick path.
    Sampling: a resumed session draws from its own key and frame count, so resume_rows switches the engine to per-row
    random streams, exactly as reset_rows(seed=...) does; sessions restore bit for bit when they were admitted with a
    seed or settings (per-row streams from the start).  Resuming into an engine of another capacity is allowed but its
    results are not promised bit for bit (the LM GEMM's split-K count depends on the batch)."""

    swap_ctas = 16
    _swap_stream: Optional[torch.cuda.Stream] = None
    # True: the LM holds a row's decoder side through its warm-up (no tokens yet), so the codec decode and the downsampler
    # run under the mask `dec_mask_dev` that `_lm_step` sets; False: under the tick's input mask
    _lm_holds_decoder = False

    def __init__(self, codec, lm, model, capacity: int, sample_rate: int, kv_pages: Optional[int], kv_page: int, n_codes: int):
        """lm: what streams with the codec (a GPT, or an LMGen); model: the LM whose scope holds the KV (the GPT, or the
        LMGen's LMModel); n_codes: the audio codes of a generated frame."""
        self.sample_rate = check_client_rate(sample_rate)
        self.frame_samples = self.sample_rate * 2 // 25                       # 80 ms at the client rate
        if capacity > MAX_STREAMS:
            raise RstnetError(f"the LM step takes at most {MAX_STREAMS} streams per scope (one weight-streaming GEMM pass), "
                              f"got {capacity}")
        self.codec, self.B, self.dev = codec, capacity, model.device
        self._lm, self._model = lm, model
        codec.streaming_forever(capacity)
        if kv_pages is None:
            lm.streaming_forever(capacity)
        else:
            lm.streaming_forever(capacity, kv_pages=kv_pages, kv_page=kv_page)
            self.kv_pages, self._kv_lm = kv_pages, model
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
        self.tok_host = torch.zeros(capacity, n_codes + 1, dtype=torch.int64, pin_memory=pin)
        self.pcm_host = torch.zeros(capacity, 1, F, dtype=torch.float32, pin_memory=pin)
        self.mask_host = torch.zeros(capacity, dtype=torch.int64, pin_memory=pin)
        self.latencies_ms: List[float] = []
        self._kv_page, self._n_codes = kv_page, n_codes
        self._row_swaps: Dict[int, torch.cuda.Event] = {}   # row -> the last gather / scatter touching it
        self._scatters: List[torch.cuda.Event] = []         # scatters the next tick waits for
        self._in_flight: List[Tuple[torch.cuda.Event, List[int]]] = []
        self._keep: List[tuple] = []                        # (event, objects a swap reads / writes, blob to pool or None)
        self._blob_pool: List[torch.Tensor] = []

    def reset_rows(self, rows, sampling=None, seed: Optional[int] = None) -> None:
        """Restart `rows`.  sampling / seed give them their own settings and random stream (keyed by the seed and the
        row's own frame count); from the first such call on, every row samples through per-row tables and keys, so a
        session's tokens do not depend on its row or its admission tick.  Until then the engine draws exactly as before.
        A session's random stream is its seed alone (None: 0): two sessions with the same settings, seed and input draw the
        same tokens, so callers that want them decorrelated pass distinct seeds."""
        if sampling is not None and not isinstance(sampling, Sampling):
            raise RstnetError(f"sampling must be a Sampling (got {type(sampling).__name__})")
        self._wait_rows(rows)
        self._reserve_first_page(rows)
        self._restart(rows, sampling, seed)

    def _restart(self, rows, sampling, seed) -> None:
        self.codec.reset_streaming(streams=list(rows))
        self._reset_lm_rows(rows, sampling, seed)
        if self.up is not None:
            self.up.reset(rows)
            self.down.reset(rows)

    @torch.no_grad()
    def step(self, pcm_rows: Dict[int, torch.Tensor], active: List[int]):
        t0 = time.perf_counter()
        self._before_tick()
        self.mask_host.zero_()
        for r, chunk in pcm_rows.items():
            self.pcm_in[r, 0].copy_(torch.as_tensor(chunk, dtype=torch.float32).reshape(self.frame_samples))
            self.mask_host[r] = 1
        self.codec.set_active_streams(self.mask_host)
        self._lm.set_active_streams(self.mask_host)
        if self.up is None:
            self.pcm_dev.copy_(self.pcm_in, non_blocking=True)
        else:
            self.up.set_active(self.mask_host)
            if not self._lm_holds_decoder:
                self.down.set_active(self.mask_host)
            self.pcm_client_dev.copy_(self.pcm_in, non_blocking=True)
            self.up(self.pcm_client_dev[:, 0], out=self.pcm_dev[:, 0])                  # r -> 24 kHz, all rows
        toks, codes, valid = self._lm_step(self.codec.encode(self.pcm_dev))     # encode: [B, 8, 1]
        if toks is not None:
            pcm = self.codec.decode(codes)                                        # [B, 1, 1920]
            if self.down is not None:
                if self._lm_holds_decoder:
                    self.down.set_active(self.dec_mask_dev)
                pcm = self.down(pcm[:, 0], out=self.pcm_out_dev)[:, None]                  # 24 kHz -> r, all rows
            self.tok_host.copy_(toks, non_blocking=True)
            self.pcm_host.copy_(pcm, non_blocking=True)
        if self.dev.type == "cuda":
            torch.cuda.current_stream(self.dev).synchronize()
        self.latencies_ms.append(1e3 * (time.perf_counter() - t0))
        return {r: (self.tok_host[r].clone(), self.pcm_host[r, 0].clone()) if valid is None or valid[r] else (None, None)
                for r in active}

    def _prune(self) -> None:
        """drop the host memory of completed swaps; the blobs of completed resumes go back to the pool"""
        keep = []
        for item in self._keep:
            if item[0].query():
                if item[2] is not None:
                    self._blob_pool.append(item[2])
            else:
                keep.append(item)
        self._keep = keep

    def _before_tick(self) -> None:
        """the tick waits for the scatters enqueued since the last one; finished swaps give back their host memory and
        pages"""
        self._wait_scatters()
        if self._keep:
            self._prune()
        if self.kv_pages is not None:
            self.reclaim()

    def pin_host_blobs(self, count: int, nbytes: int) -> None:
        """Add `count` pinned blobs of `nbytes` bytes to the pool suspensions draw from (row_bytes(positions) gives a
        session's size), so that suspending allocates no pinned memory while the engine serves."""
        for _ in range(int(count)):
            self._blob_pool.append(torch.empty(max(int(nbytes), 1), dtype=torch.uint8, pin_memory=True))

    def drop_host_blobs(self) -> None:
        """Free the pooled blobs (blobs of live SessionStates are not pooled)."""
        self._prune()
        self._blob_pool = []

    def _take_blob(self, nbytes: int) -> torch.Tensor:
        fit = [i for i, b in enumerate(self._blob_pool) if b.numel() >= nbytes]
        if fit:
            return self._blob_pool.pop(min(fit, key=lambda i: self._blob_pool[i].numel()))
        return torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)

    def row_bytes(self, positions: int) -> int:
        """the blob size of a session that has run `positions` LM positions"""
        c = self._model.config
        kv = c.n_layer * 2 * c.n_query_groups * min(int(positions), c.context) * c.head_size * 2
        return row_state.layout(self._row_regions(0, dict(self._row_host(0), pos=0)))[1] + -(-kv // row_state.ALIGN) * row_state.ALIGN

    def _side(self) -> torch.cuda.Stream:
        if self._swap_stream is None:
            self._swap_stream = torch.cuda.Stream(device=self.dev)
        return self._swap_stream

    def _wait_rows(self, rows) -> None:
        """the main stream waits for the gathers and scatters still touching these rows"""
        for r in rows:
            ev = self._row_swaps.pop(int(r), None)
            if ev is not None:
                torch.cuda.current_stream(self.dev).wait_event(ev)

    def _wait_scatters(self) -> None:
        if self._scatters:
            main = torch.cuda.current_stream(self.dev)
            for ev in self._scatters:
                main.wait_event(ev)
            self._scatters = []

    def session_key(self) -> Tuple:
        """what a SessionState must match to restore here: engine kind, LM and codec shapes, client rate, KV page"""
        cfg = self._model.config
        cfg = sorted((vars(cfg) if not hasattr(cfg, "__dataclass_fields__") else
                      {k: getattr(cfg, k) for k in cfg.__dataclass_fields__}).items())
        m = self.codec
        codec = (m.sample_rate, m.n_filters, tuple(m.ratios), m.compress, m.latent_dim, m.codebook_size, m.codebook_dim, m.n_q,
                 m.num_heads, m.num_layers, m.context)
        page = self._kv_lm._paged().pages.page if self.kv_pages is not None else self._kv_page
        return (type(self).__name__, repr(cfg), codec, self.sample_rate, page)

    def _common_regions(self, row: int, positions: int):
        regions = [("codec." + n, sg) for n, sg in self.codec._stream_state.row_segments(row, FRAME_SAMPLES, 1, self._n_codes)]
        if self.up is not None:
            regions += [("up." + n, sg) for n, sg in self.up.row_segments(row, self.frame_samples)]
            regions += [("down." + n, sg) for n, sg in self.down.row_segments(row, FRAME_SAMPLES)]
        regions += [("lm." + n, sg) for n, sg in self._model._state.row_segments(row, positions)]
        return regions

    @torch.no_grad()
    def suspend_rows(self, rows, ctas: Optional[int] = None) -> List[row_state.SessionState]:
        """Pack each row's state into a pinned host blob (one gather per row on the side stream, after the ticks already
        enqueued) and free the row: it stays held, and on a paged engine its pages return to the pool once the gather
        has completed.  -> one SessionState per row.  The caller no longer steps these rows (a FrameScheduler frees
        them); they are restarted by reset_rows or resume_rows."""
        rows = [int(r) for r in rows]
        if len(set(rows)) != len(rows) or any(not 0 <= r < self.B for r in rows):
            raise RstnetError(f"rows must be distinct and in [0, {self.B})")
        # every row's segments first (this may build the codec plans or resampler buffers, on the main stream), so that a
        # row that cannot be listed raises before anything changes, and the gathers are ordered after those writes
        key, plans = self.session_key(), []
        for r in rows:
            host = self._row_host(r)
            regions = self._row_regions(r, host)
            table, nbytes = row_state.layout(regions)
            plans.append((r, host, row_state.signature(regions), table, nbytes))
        if self._keep:
            self._prune()
        main, side = torch.cuda.current_stream(self.dev), self._side()
        side.wait_stream(main)
        states = []
        for r, host, sig, table, nbytes in plans:
            blob = self._take_blob(nbytes)
            tab = row_state.pinned_table(table)
            row_state.run("gather", tab, len(table), blob, side, ctas or self.swap_ctas)
            done = torch.cuda.Event()
            done.record(side)
            self._row_swaps[r] = done
            self._keep.append((done, (tab, blob), None))    # the gather writes the blob: alive until it completed
            states.append(row_state.SessionState(key, sig, blob, nbytes, host, done, tab))
            if self.kv_pages is not None:
                st = self._kv_lm._paged()
                self._in_flight.append((done, st.pages.detach(r)))
                st.upload_pages([r])          # stream-ordered: later ticks write nothing to the pages of this row
        return states

    @torch.no_grad()
    def resume_rows(self, rows, states, ctas: Optional[int] = None) -> None:
        """Unpack each state into its row (a free row: on a paged engine, one that holds no pages).  A paged engine first
        reserves pages for the state's positions (a short pool raises and changes nothing).  The scatter runs on the
        side stream after the ticks already enqueued and after the state's gather; the next tick waits for it.  An
        incompatible state (other engine kind, LM or codec shapes, client rate or KV page) raises RstnetError."""
        rows = [int(r) for r in rows]
        states = list(states)
        if len(rows) != len(states) or len(set(rows)) != len(rows) or any(not 0 <= r < self.B for r in rows):
            raise RstnetError(f"rows must be distinct, in [0, {self.B}), one per state")
        key = self.session_key()
        for s in states:
            if not isinstance(s, row_state.SessionState):
                raise RstnetError(f"expected a SessionState, got {type(s).__name__}")
            if s.key != key:
                row_state.check_compatible(s, key, ())
            if s.blob is None:
                raise RstnetError("this session state was already resumed")
        if len({id(s) for s in states}) != len(states):
            raise RstnetError("a session state is listed twice")
        if self.kv_pages is not None:
            pages = self._kv_lm._paged().pages
            if any(pages.held[r] for r in rows):
                raise RstnetError("resume_rows needs free rows: a listed row holds KV pages")
            self.reclaim()
            # positions up to the page boundary (at least the first page), as growth and admission reserve
            P = pages.page
            self._kv_lm.reserve_kv(rows, [max(P, -(-s.positions // P) * P) for s in states])
        try:
            plans = []
            for r, s in zip(rows, states):
                regions = self._row_regions(r, s.host)
                row_state.check_compatible(s, key, regions)
                plans.append(row_state.layout(regions)[0])
        except Exception:
            if self.kv_pages is not None:
                self._kv_lm.release_kv(rows)
            raise
        self._per_row_sampling()              # before the scatters: a first switch rewrites every row's key
        if self._keep:
            self._prune()
        main, side = torch.cuda.current_stream(self.dev), self._side()
        side.wait_stream(main)
        for r, s, table in zip(rows, states, plans):
            if s.ready is not None:
                side.wait_event(s.ready)
            prev = self._row_swaps.get(r)
            if prev is not None:
                side.wait_event(prev)
            tab = row_state.pinned_table(table)
            row_state.run("scatter", tab, len(table), s.blob, side, ctas or self.swap_ctas)
            done = torch.cuda.Event()
            done.record(side)
            self._scatters.append(done)
            self._row_swaps[r] = done        # a reset_rows of this row before the next tick waits for it too
            # the scatter reads the blob (and the gather's table may still be referenced): kept until it completed, then
            # the blob joins the pool and the state is consumed
            self._keep.append((done, (tab, s._table), s.blob))
            s.blob, s._table = None, None
            self._set_row_host(r, s.host)


class DuplexEngine(_DuplexCore):
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
        super().__init__(codec, gpt, gpt, capacity, sample_rate, kv_pages, kv_page, gpt.config.dep_q)
        self.gpt = gpt
        self.sampling = dict(use_sampling=use_sampling, temp_text=temp_text, top_k_text=top_k_text, temp=temp, top_k=top_k)
        if top_p_text or top_p:
            self.sampling.update(top_p_text=top_p_text, top_p=top_p)
        self._defaults = (use_sampling, temp_text, top_k_text, top_p_text, temp, top_k, top_p)
        self.row_sampling: Optional[List[Sampling]] = None   # per-row settings once a session brought its own
        self.row_keys = np.zeros(capacity, dtype=np.int64)
        self._keys_dirty = False
        self._valid_table = None
        self.prev_text = torch.full((capacity, 1, 1), gpt.text_initial_token_id, dtype=torch.int64, device=self.dev)

    # ---- the row state of suspend_rows / resume_rows (_DuplexCore)
    def _row_host(self, r: int) -> dict:
        return {"pos": int(self.gpt._state.pos_host[r]), "key": int(self.row_keys[r]),
                "sampling": None if self.row_sampling is None else self.row_sampling[r]}

    def _row_regions(self, r: int, host: dict):
        return self._common_regions(r, host["pos"]) + [("prev_text", row_state.tensor_segs(self.prev_text[r]))]

    def _per_row_sampling(self) -> None:
        if self.row_sampling is None:
            self.row_sampling = [Sampling(*self._defaults)] * self.B

    def _set_row_host(self, r: int, host: dict) -> None:
        self.gpt._state.pos_host[r] = host["pos"]
        self.row_sampling[r] = host["sampling"] if host["sampling"] is not None else Sampling(*self._defaults)
        self.row_keys[r] = host["key"]
        self._keys_dirty = True

    def reset_rows(self, rows, sampling=None, seed: Optional[int] = None, prompts=None) -> None:
        """_DuplexCore.reset_rows; prompts are a Moshi engine's (MoshiDuplexEngine.reset_rows): here they raise and change
        nothing."""
        if prompts is not None:
            raise RstnetError("prompts are a MoshiDuplexEngine feature: the GPT duplex engine starts sessions empty")
        super().reset_rows(rows, sampling, seed)

    def _reset_lm_rows(self, rows, sampling, seed) -> None:
        if sampling is not None or seed is not None or self.row_sampling is not None:
            default = Sampling(*self._defaults)
            if self.row_sampling is None:
                self.row_sampling = [default] * self.B
            for r in rows:
                self.row_sampling[r] = sampling if sampling is not None else default
                self.row_keys[r] = int(seed or 0) & 0xFFFFFFFF
            self._keys_dirty = True
        self.gpt.reset_streaming(streams=list(rows))
        self.prev_text[list(rows)] = self.gpt.text_initial_token_id

    def _lm_step(self, codes):
        """-> (tokens [B, dep_q + 1], the codes to decode [B, dep_q, 1], None: every row has tokens)"""
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
        return toks, toks[:, 1:, None].clamp(max=self.codec.codebook_size - 1), None


class MoshiDuplexEngine(_DuplexCore):
    """The serving loop of server.py:128-136 -- `mimi.encode -> lm_gen.step(codes) -> mimi.decode(tokens[:, 1:])` --
    for `capacity` sessions in one streaming scope of a MimiCodec and an `LMGen` (rstnet_b200.moshi).

    Every session has its own warm-up: `LMGen` returns no tokens for a row's first `max_delay` steps, and for those steps
    the codec's decoder is held for that row (the reference does not call `mimi.decode` then) while its encoder advances.
    `step` returns {row: (tokens, pcm)}, tokens = int64 [dep_q + 1] (text token, then the audio codes that were decoded),
    pcm = float32 [sample_rate * 0.08]; a row in its warm-up gets (None, None), as the reference's `lm_gen.step` returns
    None.  Text-piece decoding and the transport stay with the caller.  `sample_rate` and `kv_pages` / `kv_page` as for
    `DuplexEngine` (the pages are the LMGen's LMModel scope's)."""

    _lm_holds_decoder = True

    def __init__(self, codec, lm_gen, capacity: int, *, sample_rate: int = CODEC_RATE, kv_pages: Optional[int] = None,
                 kv_page: int = KV_PAGE):
        lm = lm_gen.lm_model
        n_user = lm.num_codebooks - lm.dep_q - 1
        if codec.n_q != n_user:
            raise RstnetError(f"the codec emits {codec.n_q} codes per frame, the LM takes {n_user} user codebooks")
        super().__init__(codec, lm_gen, lm, capacity, sample_rate, kv_pages, kv_page, lm.dep_q)
        self.lm_gen = lm_gen
        self._prefill: list = []      # LMGen._prompt_begin work lists of the rows still prefilling
        self.dec_mask_host = torch.zeros(capacity, dtype=torch.int64, pin_memory=self.dev.type == "cuda")
        self.dec_mask_dev = torch.zeros(capacity, dtype=torch.int64, device=self.dev)

    # ---- the row state of suspend_rows / resume_rows (_DuplexCore): the decoder's warm-up is the delay cache's step
    # count (off_host: no tokens, and the codec decoder held, for the first max_delay steps)
    def _row_host(self, r: int) -> dict:
        g = self.lm_gen
        return {"pos": int(g._st.lm.pos_host[r]), "off": int(g._st.off_host[r]), "stepped": bool(g._st.stepped[r]),
                "sampling": None if g._row_sampling is None else g._row_sampling[r]}

    def _row_regions(self, r: int, host: dict):
        return self._common_regions(r, host["pos"]) + [("gen." + n, sg) for n, sg in self.lm_gen._st.row_segments(r)]

    def _per_row_sampling(self) -> None:
        if self.lm_gen._row_sampling is None:
            self.lm_gen.set_stream_sampling([])

    def _set_row_host(self, r: int, host: dict) -> None:
        g = self.lm_gen
        g._st.lm.pos_host[r] = host["pos"]
        g._st.off_host[r], g._st.stepped[r] = host["off"], host["stepped"]
        g._row_sampling[r] = host["sampling"] if host["sampling"] is not None else g.default_sampling()

    # ---- prompted sessions
    def check_prompt(self, prompt) -> int:
        """-> P of a prompt int64 [K, P] in LMGen's step layout; raises RstnetError on another shape or dtype"""
        K = self.lm_gen.lm_model.num_codebooks
        if not torch.is_tensor(prompt) or prompt.dim() != 2 or prompt.shape[0] != K or prompt.dtype.is_floating_point \
                or prompt.dtype == torch.bool:
            raise RstnetError(f"a prompt is an integer tensor [{K}, P], got "
                              f"{tuple(prompt.shape) if torch.is_tensor(prompt) else type(prompt).__name__}")
        return int(prompt.shape[1])

    def reset_rows(self, rows, sampling=None, seed: Optional[int] = None, prompts=None) -> None:
        """Restart `rows` (_DuplexCore.reset_rows).  prompts {row: int64 [K, P]} (LMGen's step layout,
        moshi.prompt_from_aligned) start those rows from their prompts: LMGen.prefill_streams after the restart, so their
        first step is the one P steps of LMGen.step with the prompt's tokens forced would have reached.  On a paged engine
        a prompted row is given pages for P + 1 positions first (all rows or none: a short pool raises and changes
        nothing).  The codec rows start from a reset state, as for any new session: the prompt's audio does not prime
        the decoder or the encoder."""
        self.start_rows(rows, sampling, seed, prompts)
        while self._prefill:
            self.prefill_chunk()

    def start_rows(self, rows, sampling=None, seed: Optional[int] = None, prompts=None) -> None:
        """reset_rows without running the prefill: the prompted rows are `prefilling` until `prefill_chunk` calls have
        run it (FrameScheduler runs one per tick); they must not step until then."""
        if sampling is not None and not isinstance(sampling, Sampling):
            raise RstnetError(f"sampling must be a Sampling (got {type(sampling).__name__})")
        rows = [int(r) for r in rows]
        prompts = {int(r): p for r, p in (prompts or {}).items()}
        if any(r not in rows for r in prompts):
            raise RstnetError("every prompted row must be one of the rows restarted")
        lens = {r: self.check_prompt(p) for r, p in prompts.items()}
        self._wait_rows(rows)
        if self._kv_lm is not None and prompts:
            # all or nothing, before anything changes: prompted rows hold P + 1 positions, the others their first page
            page = self._kv_lm._paged().pages.page
            self._kv_lm.reserve_kv(rows, [lens[r] + 1 if r in lens else page for r in rows])
        self.drop_prefill(rows)
        if not prompts:
            self._reserve_first_page(rows)
        self._restart(rows, sampling, seed)
        if prompts:
            self._prefill += self.lm_gen._prompt_begin(prompts)

    @property
    def prefilling(self) -> frozenset:
        """Rows whose prompt prefill has chunks left to run."""
        return frozenset(it[0] for it in self._prefill)

    def prefill_chunk(self) -> None:
        """Run one ragged chunk (at most MAX_ROWS rows) of the pending prompt prefills, oldest first."""
        if self._prefill:
            self._prefill = self.lm_gen._prompt_chunk(self._prefill)

    def drop_prefill(self, rows) -> None:
        """Forget the pending prefill of `rows` (a session released before its prompt was in)."""
        rows = set(int(r) for r in rows)
        self._prefill = [it for it in self._prefill if it[0] not in rows]

    def _reset_lm_rows(self, rows, sampling, seed) -> None:
        self.lm_gen.reset_streaming(streams=list(rows))
        if sampling is not None or seed is not None or getattr(self.lm_gen, "_row_sampling", None) is not None:
            self.lm_gen.set_stream_sampling(list(rows), sampling, seed)

    def _lm_step(self, codes):
        """-> (tokens [B, dep_q + 1], the codes to decode [B, dep_q, 1], the rows past their warm-up), or no tokens and
        no codes while every row is in its warm-up"""
        toks = self.lm_gen.step(codes)                                           # [B, dep_q + 1, 1] or None
        valid = self.lm_gen.valid_rows()                                         # host mirror: no device sync
        if toks is None:
            return None, None, valid
        # rows in their warm-up keep their decoder state: decode mask = active & valid, a device-to-device copy
        self.dec_mask_host.copy_(torch.from_numpy(valid.astype("int64")))
        self.dec_mask_dev.copy_(self.dec_mask_host, non_blocking=True)
        self.codec.set_active_streams(self.dec_mask_dev)
        return toks[:, :, 0], toks[:, 1:].clamp(0, self.codec.codebook_size - 1), valid


class TTSEngine:
    """Request-driven streaming TTS: the batch TTS loop of InferenceImp.generate_many (`infer._TTSRows`, shared with
    stream_many) over one LM scope of `capacity` rows and one codec streaming scope, taking requests while it runs.

    `submit(utt_id, seq)` checks the request's TTS layout (InferenceImp._layout) and queues it; every `step()` admits
    queued requests in submission order into free rows (waiting for KV pages as generate_many does), runs one generated
    frame with its codec frame for all rows, and returns the chunks of the frame before it as TTSChunk(utt_id, index,
    pcm [1920] float32 on the host, codes): an utterance of G frames gives chunks 0 .. G-2, and its last chunk carries
    its codes [8, G-1] on the host, equal to generate_many's.  The host waits only for that previous frame's PCM copy,
    so the device always has the current frame queued.  `step()` with nothing admitted or queued returns [] and launches
    nothing.  The engine holds the model's and the codec's streaming scopes until `close()` (or the end of a `with`)."""

    def __init__(self, imp, codec, capacity: int, *, kv_pages: Optional[int] = None, n_samples: int = 1):
        """n_samples > 1 raises: a streamed chunk cannot wait for the ranking of best-of-N candidates."""
        from contextlib import ExitStack
        from .infer import _TTSRows, _tts_scope
        if isinstance(capacity, bool) or not isinstance(capacity, (int, np.integer)):
            raise RstnetError(f"capacity must be an int (got {capacity!r})")
        imp._check_many(int(capacity), kv_pages, n_samples, streamed=True)
        self.imp, self.codec, self.capacity = imp, codec, int(capacity)
        self._stack = ExitStack()
        try:
            self._stack.enter_context(_tts_scope(imp.model, self.capacity, kv_pages))
            self._stack.enter_context(codec.streaming(self.capacity, clip_window=True))
            self._rows = _TTSRows(imp, self.capacity, False, {}, codec)
        except BaseException:
            self._stack.close()
            raise
        self._queue: Deque[tuple] = deque()
        self._live: set = set()          # utt ids submitted whose last chunk has not been returned
        self._closed = False

    def submit(self, utt_id, seq: torch.Tensor, sampling: Optional[Sampling] = None, seed: int = 0, *,
               task: str = "TTS", lengths: Optional[Tuple[int, int]] = None) -> None:
        """Queue one utterance, seq [9, L] in the layout of `task` (TTS or audio_only; raises at once on a text task, a bad
        layout, a request longer than the whole KV pool and on an id still in flight).  sampling: its own settings (from
        then on every row samples through the per-row tables); seed: its random stream; lengths: (min_frames,
        max_frames), its window as in InferenceImp.generate_many -- an utterance that stops ends with an empty chunk
        carrying its codes (InferenceImp.stream_many)."""
        if self._closed:
            raise RstnetError("the engine is closed")
        if sampling is not None and not isinstance(sampling, Sampling):
            raise RstnetError(f"sampling must be a Sampling (got {type(sampling).__name__})")
        if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)):
            raise RstnetError(f"seed must be an int (got {seed!r})")
        if utt_id in self._live:
            raise RstnetError(f"utterance {utt_id!r} is already queued or generating")
        seq = torch.as_tensor(seq)
        if seq.dim() != 2 or seq.shape[0] != self._rows.dep_q + 1:
            raise RstnetError(f"seq must be [{self._rows.dep_q + 1}, L], got {tuple(seq.shape)}")
        req = self.imp._request(utt_id, seq, sampling, int(seed), task, lengths)
        self.imp._check_streamed(req)
        self._rows.fits(utt_id, req.P, req.G)
        if sampling is not None:
            self._rows.use_per_row()
        self._live.add(utt_id)
        self._queue.append(req)

    @property
    def pending(self) -> int:
        """requests submitted and not yet admitted"""
        return len(self._queue) + (self._rows.pending is not None)

    @property
    def active(self) -> int:
        """admitted utterances whose last chunk has not been returned yet"""
        return len(self._live) - self.pending

    @torch.no_grad()
    def step(self) -> List:
        if self._closed:
            raise RstnetError("the engine is closed")
        chunks = self._rows.stream_step(lambda: self._queue.popleft() if self._queue else None) or []
        for c in chunks:
            if c.codes is not None:
                self._live.discard(c.utt_id)
        return chunks

    def close(self) -> None:
        """Leave the scopes (the chunks of a frame still in flight are dropped) and check the LM's device error flags."""
        if self._closed:
            return
        self._closed = True
        try:
            if self._rows.n:
                self.imp.model.check_device_errors()
        finally:
            self._stack.close()

    def __enter__(self) -> "TTSEngine":
        return self

    def __exit__(self, *exc) -> None:
        self.close()
