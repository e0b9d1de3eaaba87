"""Streaming O(1)-per-frame version of the reference's offline generation loop.

Mirrors ``InferenceImp`` and ``reverse_delay`` of MLLM_v2/infer_no_streaming.py:149-323 (same constructor and call
signature, same special token ids, same per-codebook sampling rules), but instead of re-running the whole prefix
through ``forward_global`` and re-running ``forward_local`` 8 times per generated frame (O(T^2) per utterance,
SURVEY.md §3.1) it streams: the prompt goes through ``GPT.prefill`` (multi-position chunks writing the KV rings in one
pass), and each generated frame is one ``GPT.forward_step`` (temporal step + 8 depth steps + device-side sampling, one
CUDA-graph replay).  The arithmetic per frame is the reference's: upstream evaluates the depth transformer through the
NON-streaming ``forward_local`` (every depth step sees all earlier keys), so ``forward_step`` runs with
``depth_ring_quirk=False`` here; the temporal transformer's non-streaming form equals the streamed one while the
sequence is shorter than ``config.context`` (tests/test_lm_gpu.py checks the loop against the reference's own tokens).
All four tasks of the reference loop run (``TASKS``; upstream only TTS returns, the other branches raise after their
loop at an unbound ``gt_audio``): each has its own layout (``InferenceImp._layout``) and a window (minlen, maxlen) with
the reference's early stop, which the device decides per row inside the frame graph (rstnet_lm_gen_rows_advance).

``InferenceImp.generate_many`` runs a corpus of utterances, each with its own prompt and generation length, as one
continuously batched scope: a row that finishes is refilled with the next utterance (ragged prefill of that row alone,
``GPT.prefill_streams``), and every row samples with its own candidate sets and random stream, so an utterance's codes do
not depend on its row, on its admission time or on the other utterances.

Mode 'teacher-force' (infer_no_streaming.py:172-182) scores a sequence instead of generating: ``InferenceImp.score_many``
packs the frames of several utterances into shared ragged chunks (the row map of ``GPT.prefill_streams``) run with the
lm_head on, and feeds each chunk's text logits, and the depth transformer's audio logits on the same rows, to the
cross-entropy kernel, which adds into one accumulator slot per utterance; ``__call__`` in that mode is score_many on one
utterance.
"""
from __future__ import annotations

from contextlib import contextmanager
from dataclasses import dataclass
from typing import Dict, Iterable, Iterator, List, NamedTuple, Optional, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import RstnetError
from .lm import GPT, KV_PAGE, MAX_STREAMS, Sampling, score_item, score_packed

TASKS = ("TTS", "audio_only", "text_only", "ASR")   # infer_no_streaming.py:184-226
AUDIO_TASKS = ("TTS", "audio_only")                 # the tasks whose generated frames are audio to stream
SEMANTIC_PAD = 2049                                 # the semantic pad id: audio_only / TTS strip trailing frames by it


def candidate_counts(pre_gen_len: int, minlen: int, g_idx: int, dep_q: int = 8) -> List[int]:
    """Candidate-set size of each codebook at generated frame g_idx (infer_no_streaming.py:264-283): 2049 ids on the first
    generated frame and for codebooks > 0 once g_len > minlen, 2048 otherwise."""
    g_len = pre_gen_len + g_idx
    return [2049 if (g_len == pre_gen_len or (l > 0 and g_len > minlen)) else 2048 for l in range(dep_q)]


SEED_STRIDE = 0x9E3779B9   # odd: i -> seed + i * SEED_STRIDE (mod 2^32) is one-to-one


def sample_seed(seed: int, i: int) -> int:
    """The random-stream key of candidate i of an utterance whose seed is `seed` (generate_many(n_samples=N)): seed + i *
    0x9E3779B9 modulo 2^32, and `seed` itself for i = 0 (the sampler reads a key modulo 2^32), so candidate 0 draws what
    the utterance draws alone.  The stride is odd, so the N keys of an utterance differ for any N <= 2^32."""
    seed, i = int(seed), int(i)
    if i < 0:
        raise RstnetError(f"a candidate index is >= 0 (got {i})")
    return seed if i == 0 else (seed + i * SEED_STRIDE) & 0xFFFFFFFF


class Candidate(NamedTuple):
    """One of the n_samples candidates of an utterance (generate_many(n_samples=N)): `index` i (its random stream is
    sample_seed(seed, i)), codes [8, G-1] (the generated frames [G, 9] for a task other than TTS), the summed
    log-probabilities of its sampled audio tokens (the 8 audio heads over all G frames) and text tokens under the model's
    untempered softmax, and its frame count G (the frames it kept, when its window stopped it)."""
    index: int
    codes: torch.Tensor
    logprob_audio: float
    logprob_text: float
    frames: int


def rank_candidates(cands: List[Candidate], rank: Optional[str]) -> List[Candidate]:
    """rank 'logprob': highest mean audio log-probability per frame first, ties by index (a candidate that stopped before
    its first frame last); None: index order"""
    if rank is None:
        return sorted(cands, key=lambda c: c.index)
    return sorted(cands, key=lambda c: (-c.logprob_audio / c.frames if c.frames else float("inf"), c.index))


def continuation_codes(seq: torch.Tensor, frames: torch.Tensor) -> torch.Tensor:
    """The clip of an audio_only item: its prompt audio (the first L // 2 frames of seq [9, L] after the pad frames are
    stripped, as _layout does) followed by its generated frames [G', 9], with the one-frame acoustic delay undone over the
    whole -> codes [8, P + G' - 1].  The prompt's last frame takes codebooks 1..7 from the first generated frame, so the
    clip decodes without a seam at the join (the reference concatenates the two, :301-302)."""
    pad_len = int(seq[1].eq(SEMANTIC_PAD).int().sum().item())
    P = (seq.shape[1] - pad_len) // 2
    audio = torch.cat([seq[1:, :P].to(frames.device, torch.int64), frames[:, 1:].t().to(torch.int64)], dim=1)
    return reverse_delay_rows(audio)


def reverse_delay_rows(x: torch.Tensor) -> torch.Tensor:
    """reverse_delay of codes already laid out [8, L] (no orientation guess: any L)"""
    out = torch.empty_like(x[:, :-1])
    out[0] = x[0, :-1]
    out[1:] = x[1:, 1:]
    return out


def reverse_delay(x: torch.Tensor) -> torch.Tensor:
    """Undo the one-frame acoustic delay (infer_no_streaming.py:311-323): x [8, L] (or [L, 8]) -> [8, L-1] with
    row 0 kept and rows 1..7 shifted left by one frame."""
    if x.shape[0] != 8:
        x = x.transpose(0, 1)
    out = torch.empty_like(x[:, :-1])
    out[0] = x[0, :-1]
    out[1:] = x[1:, 1:]
    return out


class InferenceImp(object):
    def __init__(self, args, model: GPT, mode, temp_text, top_k_text, temp, top_k, task_name):
        self.model, self.args = model, args
        self.n_samples = 1
        self.task_name = task_name
        self.text_pad_token = 128003
        self.acoustic_pad_token = 2049
        self.semantic_pad_token = SEMANTIC_PAD
        self.text_empty_token = 128002
        self.mode = mode
        self.use_sampling = True          # upstream hard-codes True (:162); set the attribute to False for argmax decoding
        self.temp_text, self.top_k_text, self.temp, self.top_k = temp_text, top_k_text, temp, top_k
        self.top_p_text, self.top_p = 0.0, 0.0   # nucleus sampling of the text / audio heads (0: off, as upstream's callers)

    def sampling(self) -> Sampling:
        """the instance's settings as one Sampling (validated)"""
        return Sampling(bool(self.use_sampling), self.temp_text, self.top_k_text, self.top_p_text, self.temp, self.top_k, self.top_p)

    @torch.no_grad()
    def __call__(self, seq: torch.Tensor, mask: torch.Tensor):
        """seq [9, L] (one utterance, as upstream) -> codes [8, T'] after reverse_delay (task 'TTS'), or the generated
        frames [G', 9] (the other tasks).  In mode 'teacher-force'
        (infer_no_streaming.py:172-182, before any padding removal or task check) -> (loss_audio / 8, loss_text) as 0-dim
        fp64 tensors: score_many on this one utterance."""
        if self.mode == "teacher-force":
            _, met = next(self.score_many([(None, seq, mask)], capacity=1))
            return (torch.tensor(met["loss_audio"], dtype=torch.float64), torch.tensor(met["loss_text"], dtype=torch.float64))
        return self.generate(seq.unsqueeze(0).expand(self.n_samples, -1, -1))[0]

    @torch.no_grad()
    def generate(self, seq: torch.Tensor, return_frames: bool = False):
        """Batched form: seq [B, 9, L], all rows in the same TTS layout (same prompt length and number of frames to
        generate; row 0 defines them, as upstream reads `seq[0]`).  -> codes [B, 8, T'] (and the raw frames [B, G, 9]).
        The other tasks: -> a list of B generated frames [G'_b, 9] (rows may stop at different frames), run by
        generate_many with row b's random stream keyed b, as this loop keys row b (return_frames raises: the frames
        are the result)."""
        self._check_task()
        if self.task_name != "TTS":
            if return_frames:
                raise RstnetError(f"task {self.task_name!r} returns its generated frames: return_frames is for TTS")
            got = dict(self.generate_many(((b, seq[b]) for b in range(seq.shape[0])), seq.shape[0],
                                          seeds={b: b for b in range(seq.shape[0])}))
            return [got[b] for b in range(seq.shape[0])]
        m = self.model
        dev = seq.device
        prefix_len, _, maxlen = self._layout(seq[0])
        prefix = seq[:, :, :prefix_len]
        minlen = maxlen
        B = prefix.shape[0]
        pre_gen_len = prefix.shape[2]
        frames = []
        with m.streaming(B):
            # the init token + all prompt frames but the last only feed the KV rings (their outputs are never sampled);
            # the step on the last prompt frame yields generated frame 0
            init = m._get_initial_token().expand(B, -1, -1).to(dev)
            feed = torch.cat([init, prefix], dim=2)
            m.prefill(feed[:, :, :-1].contiguous())
            cur = feed[:, :, -1:].contiguous()
            for g_idx in range(maxlen):
                g_len = pre_gen_len + g_idx
                # per-codebook candidate sets (infer_no_streaming.py:264-283): 2049 ids on the first generated frame
                # and for codebooks > 0 once g_len > minlen, otherwise 2048
                valid = tuple(candidate_counts(pre_gen_len, minlen, g_idx))
                toks = m.forward_step(cur, use_sampling=self.use_sampling, temp_text=self.temp_text, top_k_text=self.top_k_text,
                                      temp=self.temp, top_k=self.top_k, audio_valid=valid, depth_ring_quirk=False,
                                      top_p_text=self.top_p_text, top_p=self.top_p)
                frames.append(toks)
                cur = toks[:, :, None]
            m.check_device_errors()
        raw = torch.stack(frames, dim=1).to(dev)                          # [B, G, 9]
        codes = torch.stack([reverse_delay(raw[b, :, 1:]) for b in range(B)], 0)
        return (codes, raw) if return_frames else codes

    def _check_task(self, task: Optional[str] = None):
        task = self.task_name if task is None else task
        if task not in TASKS:
            raise NotImplementedError(f"task {task!r}: the reference loop runs {', '.join(TASKS)} (infer_no_streaming.py:184-226)")
        if self.mode == "teacher-force":
            raise NotImplementedError("teacher-force mode scores sequences (__call__ / score_many), it does not generate")

    def _score_item(self, seq, mask) -> Tuple[torch.Tensor, torch.Tensor, int]:
        """Host-side checks of one scoring item -> (seq int64 [9, L], mask fp32 [9, L], frames to score) (lm.score_item):
        trailing all-zero-mask frames are dropped, and at most `context` frames remain."""
        m = self.model
        return score_item(seq, mask, m.config.n_q + 1, max_frames=m.config.context)

    def _score_metrics(self, sums_audio: torch.Tensor, sums_text: torch.Tensor, frames: int) -> dict:
        from .lm import combine_sums
        dep_q = sums_audio.shape[0]
        a, t = combine_sums(sums_audio, [1] * dep_q), combine_sums(sums_text, [1])
        return {"frames": frames, "loss_audio": float(a["loss"]) / dep_q, "loss_text": float(t["loss"]),
                "acc_all_audio": float(a["acc_all"]), "acc_target_audio": float(a["acc_target"]),
                "acc_all_text": float(t["acc_all"]), "acc_target_text": float(t["acc_target"]),
                "sums_audio": sums_audio.tolist(), "sums_text": sums_text.tolist()}

    @torch.no_grad()
    def score_many(self, items: Iterable[Tuple[object, torch.Tensor, torch.Tensor]], capacity: int = 8) -> Iterator[Tuple]:
        """Teacher-forced scoring (infer_no_streaming.py --inference_mode teacher-force) of (utt_id, seq [9, L], mask [9, L])
        items: yields (utt_id, metrics) in completion order.  metrics: loss_audio (the reference's loss_audio / 8: the mean
        over the codebooks of sum(mask * nll) / #(mask != 0), ignore id 2049), loss_text (ignore id 128003), acc_all /
        acc_target of audio and text, frames scored and the per-codebook sums sums_audio [8][5], sums_text [1][5] (fields
        lm.CE_FIELDS).  A group whose mask is zero throughout gives NaN, as upstream.

        Up to `capacity` utterances are live, one stream each; their frames are packed into ragged chunks of at most
        MAX_ROWS rows (GPT.prefill_streams' row map) run with the lm_head on; each chunk's rows go to the text
        cross-entropy, through the depth transformer on the same rows, and to the audio cross-entropy, whose sums land in
        the utterance's own accumulator slot.  No [L, V] logits are kept."""
        if not 1 <= capacity <= MAX_STREAMS:
            raise RstnetError(f"capacity must be in [1, {MAX_STREAMS}] (got {capacity})")
        m = self.model
        with m.streaming(capacity):
            for utt, sa, stx, L in score_packed(m, m._state, items, capacity, self.text_pad_token, self.acoustic_pad_token,
                                                "labels", self._score_item):
                yield utt, self._score_metrics(sa, stx, L)

    def _layout(self, seq: torch.Tensor, task: Optional[str] = None) -> Tuple[int, int, int]:
        """seq [9, L] -> (prompt length P, minlen, maxlen) of `task` (default the instance's) after stripping the pad
        frames (infer_no_streaming.py:184-226):
          * text_only / ASR strip as many trailing frames as row 0 holds text pads, audio_only / TTS as many as row 1
            holds semantic pads;
          * text_only / audio_only: P = L // 2, minlen = maxlen = P;
          * TTS: P = L - G with G the text-empty frames, minlen = maxlen = G;
          * ASR: with e text-empty frames, P = e + 1 (at most L), maxlen = L - e + 13, minlen = L - e - 13.
        At most maxlen frames are generated; from g_idx > minlen on, a frame with an id >= 2048 in audio codebooks 3..7
        ends the utterance and is dropped, so an utterance whose maxlen - 1 <= minlen always runs maxlen frames."""
        task = self.task_name if task is None else task
        self._check_task(task)
        pad_row, pad = (0, self.text_pad_token) if task in ("text_only", "ASR") else (1, self.semantic_pad_token)
        L = seq.shape[1] - int(seq[pad_row].eq(pad).int().sum().item())
        if task in ("text_only", "audio_only"):
            if L < 2:
                raise RstnetError(f"a {task} item needs 2 frames or more after its pad frames (got {L})")
            return L // 2, L // 2, L // 2
        empty = int(seq[0, :max(L, 0)].eq(self.text_empty_token).int().sum().item())
        if task == "ASR":
            if L < 1:
                raise RstnetError("the ASR item has no frames after its pad frames")
            return min(empty + 1, L), L - empty - 13, L - empty + 13
        prefix_len = L - empty
        if L - prefix_len <= 0:
            raise RstnetError("nothing to generate: the sequence has no text-empty frames")
        if prefix_len <= 0:
            raise RstnetError("the sequence has no prompt frames")
        return prefix_len, L - prefix_len, L - prefix_len

    def _request(self, utt, seq, sp, seed, task=None, lengths=None) -> "_Request":
        task = self.task_name if task is None else task
        P, minlen, maxlen = self._layout(seq, task)
        if lengths is not None:
            if (not isinstance(lengths, (tuple, list)) or len(lengths) != 2
                    or not all(isinstance(v, (int, np.integer)) and not isinstance(v, bool) for v in lengths)):
                raise RstnetError(f"lengths[{utt!r}] is (min_frames, max_frames), two ints (got {lengths!r})")
            minlen, maxlen = int(lengths[0]), int(lengths[1])
            if not 1 <= maxlen < 2 ** 31 or not -2 ** 31 <= minlen < 2 ** 31:
                raise RstnetError(f"lengths[{utt!r}]: max_frames must be in [1, 2^31) and min_frames an int32 (got {lengths!r})")
        return _Request(utt, seq, P, maxlen, sp, seed, task, minlen, maxlen - 1 > minlen)

    def _check_forced(self, utt, forced, G: int) -> np.ndarray:
        """forced[utt]: int64 [dep_q + 1, G] over the item's G generated frames, each id -1 (sample) or inside its head's
        vocabulary -> the host int32 table the frame loop reads"""
        c = self.model.config
        n_cb = self.model.num_codebooks
        if not torch.is_tensor(forced) or forced.dtype != torch.int64 or tuple(forced.shape) != (n_cb, G):
            raise RstnetError(f"forced[{utt!r}] must be an int64 tensor [{n_cb}, {G}] (its generated frames; -1: sample), got "
                              f"{(tuple(forced.shape), forced.dtype) if torch.is_tensor(forced) else type(forced).__name__}")
        f = forced.cpu().numpy()
        vocab = np.array([c.padded_vocab_size] + [c.audio_card] * (n_cb - 1))[:, None]
        if ((f < -1) | (f >= vocab)).any():
            raise RstnetError(f"forced[{utt!r}]: every id is -1 or inside its head's vocabulary (text < {c.padded_vocab_size}, "
                              f"audio < {c.audio_card})")
        return f.astype(np.int32)

    def _check_many(self, capacity: int, kv_pages: Optional[int], n_samples: int = 1, streamed: bool = False) -> None:
        """the argument checks of generate_many / stream_many / serve.TTSEngine"""
        self._check_task()
        if streamed and self.task_name not in AUDIO_TASKS:
            raise NotImplementedError(f"streamed generation runs {AUDIO_TASKS} (the instance's task is {self.task_name!r})")
        if not 1 <= capacity <= MAX_STREAMS:
            raise RstnetError(f"capacity must be in [1, {MAX_STREAMS}] (got {capacity})")
        if not hasattr(self.model, "reserve_kv") and kv_pages is not None:
            raise RstnetError(f"{type(self.model).__name__} has no paged KV scope (kv_pages)")
        if isinstance(n_samples, bool) or not isinstance(n_samples, (int, np.integer)) or n_samples < 1:
            raise RstnetError(f"n_samples must be an int >= 1 (got {n_samples!r})")
        if n_samples > 1:
            if streamed:
                raise RstnetError("streamed TTS takes n_samples = 1: a chunk is handed out before the candidates are ranked")
            if n_samples > capacity:
                raise RstnetError(f"n_samples = {n_samples} candidates need as many rows, more than capacity = {capacity}")
            if not hasattr(self.model, "fork_kv"):
                raise RstnetError(f"{type(self.model).__name__} has no paged KV scope to fork a prompt into n_samples rows")

    @staticmethod
    def _check_streamed(req: "_Request") -> None:
        """streamed generation runs the audio tasks (their generated frames decode to audio)"""
        if req.task not in AUDIO_TASKS:
            raise RstnetError(f"utterance {req.utt!r}: task {req.task!r} generates text; streamed generation runs {AUDIO_TASKS}")

    @staticmethod
    def _check_forced_keys(forced: dict, utts) -> None:
        unknown = [u for u in forced if u not in utts]
        if unknown:
            raise RstnetError(f"forced names utterance(s) that are not among the items: {unknown[:5]!r}")

    @staticmethod
    def _check_sampling(sampling: Optional[Dict[object, Sampling]]) -> None:
        if sampling is not None:
            for utt, sp in sampling.items():
                if not isinstance(sp, Sampling):
                    raise RstnetError(f"sampling[{utt!r}] must be a Sampling (got {type(sp).__name__})")

    def _puller(self, items, seeds, sampling, tasks=None, lengths=None, streamed=False, forced=None, tables=None):
        """-> pull(): the next item of `items` as an admission request (_request), or None once they are exhausted; items
        are read one at a time, when a row can take them.  streamed: the text tasks raise (their frames are no audio).
        forced: each request's forced table is checked (_check_forced) into `tables` {utt_id: int32 [9, G]}; a table for
        an utterance that is not among the items raises, before any launch when `items` is a list or tuple, else once they
        are exhausted."""
        source, seeds, done = iter(items), seeds or {}, []
        tasks, lengths, forced = tasks or {}, lengths or {}, forced or {}
        if forced and isinstance(items, (list, tuple)):
            self._check_forced_keys(forced, {it[0] for it in items})
        seen = set()

        def pull():
            if done:
                return None
            try:
                utt, seq = next(source)
            except StopIteration:
                done.append(True)
                if forced:
                    self._check_forced_keys(forced, seen)
                return None
            if forced:
                seen.add(utt)
            req = self._request(utt, seq, None if sampling is None else sampling.get(utt), int(seeds.get(utt, 0)),
                                tasks.get(utt, self.task_name), lengths.get(utt))
            if utt in forced:
                tables[utt] = self._check_forced(utt, forced[utt], req.G)
            if streamed:
                self._check_streamed(req)
            return req
        return pull

    @torch.no_grad()
    def generate_many(self, items: Iterable[Tuple[object, torch.Tensor]], capacity: int,
                      seeds: Optional[Dict[object, int]] = None, return_frames: bool = False,
                      sampling: Optional[Dict[object, Sampling]] = None, kv_pages: Optional[int] = None,
                      stats: Optional[dict] = None, n_samples: int = 1, rank: Optional[str] = "logprob",
                      tasks: Optional[Dict[object, str]] = None,
                      lengths: Optional[Dict[object, Tuple[int, int]]] = None,
                      forced: Optional[Dict[object, torch.Tensor]] = None) -> Iterator[Tuple]:
        """Continuous batching over (utt_id, seq [9, L]) items, each in its own TTS layout: yields (utt_id, codes [8, G-1])
        in completion order.  Up to `capacity` utterances decode together, one graph replay per frame; a finished row is
        held until the next utterance is admitted into it (its prompt fed through GPT.prefill_streams while the other
        rows keep their state).  Each utterance samples with its own candidate sets (candidate_counts) and its own random
        stream, keyed by seeds[utt_id] (default 0) and its own frame count from 0: with the defaults its codes are those
        of generate() on that utterance alone.  return_frames: yield (utt_id, codes, raw frames [G, 9]) as generate does.
        sampling: {utt_id: Sampling} gives those utterances their own settings (the others take the instance's); each
        utterance's codes are then those of generate() on it alone with its settings, whatever the others' settings.
        The settings are rows of device tables: changing them captures no new graph.

        The KV cache is paged (GPT.streaming(B, kv_pages=N)): an admitted utterance holds pages for exactly the positions
        it writes (its prompt and init token feed, then one per generated frame) and frees them when it finishes.
        kv_pages: the pool size in pages of lm.KV_PAGE positions; None gives every row a whole ring (capacity x
        ceil(context / KV_PAGE) pages), so admissions and completion order are those of unpaged rings.  With a smaller
        pool an utterance waits for pages while a row is free; admission stops at the first utterance that does not fit,
        so the completion order is fixed for a given pool.  An utterance needing more than the whole pool raises.
        stats: a dict that receives 'frames' (frames run), 'row_frames' (occupied rows summed over frames) and
        'wait_frames' (frames run while an utterance waited for pages with a row free).

        n_samples N > 1 (best-of-N): each utterance is N candidates in N rows, admitted together once N rows and their
        pages are free.  Its prompt is prefilled into one row and forked into the others (GPT.fork_kv): the candidates
        share the prompt's full KV pages and hold private pages only for what they write (a shared page is copied when a
        candidate reaches it again at a ring wrap).  Candidate i samples with the utterance's settings and the random
        stream sample_seed(seed, i), so its codes are those of the utterance alone with that seed.  The frames run with
        logprob=True: each candidate's sampled tokens' log-probabilities are summed on the device.  Yields (utt_id,
        [Candidate]) per utterance, ranked by `rank`: 'logprob' highest mean audio log-probability per frame first (ties
        by index), None index order.  return_frames is not available there.

        tasks: {utt_id: task} runs those items as another of TASKS than the instance's task_name, in that task's layout
        (_layout); an item of a task other than TTS yields (utt_id, frames [G', 9]): its generated frames (text token,
        audio codebooks 0..7), as the reference builds them (the text row of its `prefix`, the audio rows of its
        `final_results`).  lengths: {utt_id: (min_frames, max_frames)} replaces an item's window (minlen, maxlen) -- on TTS
        the open-length mode: at most max_frames frames, and from frame min_frames + 1 on the reference's stop rule (an id
        >= 2048 in audio codebooks 3..7; that frame is dropped).  A row whose window can stop is decided on the device
        (rstnet_lm_gen_rows_advance in the frame graph); the host reads frame n's statuses after it has enqueued frame
        n + 1, so such a row runs one frame past its stop before it is released.  It reserves KV pages for P + max_frames
        positions: that extra frame is at most frame max_frames - 1.  With no such row in the batch, no status is read.

        forced: {utt_id: int64 [9, G]} fixes tokens of an utterance's generated frames, G its maxlen: column g is generated
        frame g (text token, audio codebooks 0..7, the layout of return_frames' frames, before reverse_delay), -1 where the
        head samples.  A forced token is the frame's token everywhere: the next depth step, the next frame's input, the
        log-probability sums and the stop rule (e.g. fix the semantic codebook 0 and sample the others).  It need not lie
        in the frame's candidate set, only in its head's vocabulary.  The candidates of one utterance (n_samples > 1)
        share its table.  Each frame the loop fills every forced row's slice of a pinned [B, 9] table from the host and
        uploads it without a synchronise; the frames run the forced graph (with -1 everywhere else, it draws what the plain
        frame draws).  Shape, dtype and ids are checked at admission, before the item is launched."""
        self._check_many(capacity, kv_pages, n_samples)
        if forced is not None and not isinstance(forced, dict):
            raise RstnetError("forced must be a dict keyed by utt_id")
        if rank not in ("logprob", None):
            raise RstnetError(f"rank is 'logprob' or None (got {rank!r})")
        if n_samples > 1 and return_frames:
            raise RstnetError("return_frames is not available with n_samples > 1")
        m = self.model
        self._check_sampling(sampling)
        tables = {} if forced else None
        pull = self._puller(items, seeds, sampling, tasks, lengths, forced=forced, tables=tables)
        with _tts_scope(m, capacity, kv_pages):
            rows = _TTSRows(self, capacity, sampling is not None, {} if stats is None else stats, n_samples=int(n_samples),
                            forced=tables)
            groups: Dict[int, list] = {}
            ready = []   # utterances whose candidates all finished in the last frame: their sums are still being copied
            while True:
                rows.admit(pull)
                last = not rows.occupied()
                done = rows.settle() if last else rows.frame()
                # the sums of the previous frame's finished candidates were copied to the host after that frame, and this
                # frame is already enqueued: reading them now keeps the device busy while the host waits for the copy
                for utt, cands in ready:
                    yield utt, _ranked(cands, rank)
                ready = []
                for utt, codes, raw, st in done:
                    result = codes if st.task == "TTS" else raw
                    group = groups.setdefault(st.group, [])
                    group.append((st, result))
                    if len(group) < n_samples:
                        continue
                    del groups[st.group]
                    if n_samples > 1:
                        ready.append((utt, group))
                    elif return_frames and st.task == "TTS":
                        yield utt, codes, raw
                    else:
                        yield utt, result
                if last:
                    break
            for utt, cands in ready:
                yield utt, _ranked(cands, rank)
            m.check_device_errors()

    @torch.no_grad()
    def stream_many(self, items: Iterable[Tuple[object, torch.Tensor]], capacity: int, codec,
                    *, seeds: Optional[Dict[object, int]] = None, sampling: Optional[Dict[object, Sampling]] = None,
                    kv_pages: Optional[int] = None, n_samples: int = 1, tasks: Optional[Dict[object, str]] = None,
                    lengths: Optional[Dict[object, Tuple[int, int]]] = None) -> Iterator["TTSChunk"]:
        """generate_many's corpus, options and admissions, with the audio streamed: every frame also undoes the TTS delay
        on the device and decodes one codec frame for each row that has one (see `_TTSRows`), and the PCM is yielded as
        TTSChunk(utt_id, index, pcm [1920] float32 on the host, codes) while the utterances are still generating.  An
        utterance of G frames gives chunks 0 .. G-2 in order (their concatenation is `codec.decode` of its codes); its
        last chunk carries its codes [8, G-1] (those generate_many yields; on the host), the others None.  G = 1 gives one
        chunk of no samples.  The host hands out frame n's chunks while the device runs frame n + 1, so chunks of
        different utterances interleave in frame order.  codec: a MimiCodec on the model's device; it runs its own
        streaming scope of `capacity` rows for the duration, with clip_window rings, so that the chunks are the utterance's
        whole-clip decode at any length.  n_samples > 1 raises: a chunk cannot wait for the candidates' ranking.

        tasks / lengths as generate_many, for the audio tasks (TTS, audio_only; a text task raises): an audio_only item
        streams its continuation, codes [8, G'-1] the delay undone over its generated frames.  A row whose window can stop
        it has each chunk handed out once its frame's status is known (one frame later than a fixed row's): the chunk of
        the frame its stop fired on, which would decode the dropped frame, is not handed out; an empty chunk at that index
        carries the codes instead, so its chunks are 0 .. G'-2 with audio and G'-1 empty.  Chunks of the frame it ran
        after its stop are dropped."""
        self._check_many(capacity, kv_pages, n_samples, streamed=True)
        self._check_sampling(sampling)
        pull = self._puller(items, seeds, sampling, tasks, lengths, streamed=True)
        with _tts_scope(self.model, capacity, kv_pages), codec.streaming(capacity, clip_window=True):
            rows = _TTSRows(self, capacity, sampling is not None, {}, codec)
            while True:
                chunks = rows.stream_step(pull)
                if chunks is None:
                    break
                yield from chunks
            self.model.check_device_errors()


class TTSChunk(NamedTuple):
    """One codec frame of streamed TTS audio: `index` counts the utterance's chunks from 0; pcm float32 [1920] (80 ms at
    24 kHz) on the host; codes: the utterance's codes [8, G-1] on its last chunk, None before."""
    utt_id: object
    index: int
    pcm: torch.Tensor
    codes: Optional[torch.Tensor]


@contextmanager
def _tts_scope(m, capacity: int, kv_pages: Optional[int]):
    """The LM scope of batch TTS: GPT decodes on paged KV (None: a whole ring per row, capacity x ceil(context / KV_PAGE)
    pages); a stand-in model that offers only the unpaged streaming protocol (no reserve_kv) runs its own scope."""
    if not hasattr(m, "reserve_kv"):
        with m.streaming(capacity):
            yield
        return
    if kv_pages is None:
        kv_pages = capacity * -(-m.config.context // KV_PAGE)
    with m.streaming(capacity, kv_pages=kv_pages):
        yield


class _Request(NamedTuple):
    """An admission request of the batch loop (InferenceImp._request): the item's prompt of P frames, G = maxlen the
    frames it may run, its Sampling (None: the instance's) and seed; windowed: its window can stop it (maxlen - 1 >
    minlen), so the device decides its status every frame."""
    utt: object
    seq: torch.Tensor
    P: int
    G: int
    sampling: Optional[Sampling]
    seed: int
    task: str
    minlen: int
    windowed: bool


@dataclass(eq=False)
class _Row:
    """The state of one occupied row of the batch loop: what it was admitted with (`g` counts the frames it has run,
    from frame `start` on; `cand` is its candidate index in request `group`), then its outcome, set when it finishes:
    its result is frames start .. end - 1; stopped: its stop rule fired on frame `end` (`dropped`, not part of the
    result); lp: (host sums, row, event or None) of its log-probability sums (best-of-N); codes: its codes (audio tasks);
    forced: the request's forced table."""
    utt: object
    P: int
    G: int
    start: int
    sampling: Optional[Sampling]
    task: str
    minlen: int
    windowed: bool
    cand: int
    group: int
    g: int = 0
    end: Optional[int] = None
    stopped: bool = False
    dropped: Optional[torch.Tensor] = None
    lp: Optional[tuple] = None
    codes: Optional[torch.Tensor] = None
    forced: Optional[np.ndarray] = None

    @property
    def frames(self) -> int:
        return self.end - self.start


class _TTSRows:
    """The admission and frame loop of batch TTS, shared by generate_many, stream_many and serve.TTSEngine, inside one LM
    scope of B rows (`_tts_scope`).  `admit(pull)` fills free rows in order with the requests pull() gives (a _Request,
    None when there is none), each as n_samples rows, and stops at the first one whose rows or KV pages are not free yet
    (it waits, in `pending`, for the next call); `frame()` runs one generated frame for every row and returns the rows it
    finished as (utt, codes [8, G-1] or None, raw frames [G, 9], row state).  per_row: every row samples with its own
    settings (a request's Sampling, else the InferenceImp's) from the per-row tables; False: the instance's scalar settings.

    With a codec (stream_step), every frame also runs, for all B rows, the acoustic-delay cache kernel
    (_TTSDelay: codec frame f = codebook 0 of generated frame f and codebooks 1-7 of frame f + 1, reverse_delay on the
    device) and one step of the codec's streaming decoder, holding the rows that have no undelayed frame (a row's first
    generated frame, free rows); the PCM goes to one of two pinned host slots, and the host waits only for the previous
    frame's copy before it hands that frame's chunks out.  No eager torch arithmetic runs on this path, except the clamp of
    the codes to the codebook (ids 2048 / 2049 are LM samples, which the codec's gather clamps alike but flags as errors)."""

    def __init__(self, imp: InferenceImp, B: int, per_row: bool, stats: dict, codec=None, n_samples: int = 1,
                 forced: Optional[dict] = None):
        m = imp.model
        self.imp, self.m, self.B, self.stats = imp, m, B, stats
        self.n_samples = n_samples      # > 1: each request is that many candidates, forked from one prefill
        self.forced = forced            # {utt: int32 [9, G]} (generate_many(forced=)): every frame runs the forced graph
        self.groups = 0                 # requests admitted (a row's group id)
        stats.update(frames=0, row_frames=0, wait_frames=0)
        self.default = None             # the instance's Sampling while rows sample with per-row settings
        if per_row:
            self.use_per_row()
        self.paged = hasattr(m, "reserve_kv")
        self.pages = m._state.pages if self.paged else None   # the scope's allocator, read to decide admissions
        self.dev, n_cb = m.device, m.num_codebooks
        self.dep_q = n_cb - 1                 # text + dep_q audio codebooks per frame
        self.rows: List[Optional[_Row]] = [None] * B
        self.history: Dict[int, torch.Tensor] = {}       # frame -> tokens [B, 9] of every row
        self.n = 0                                       # frames run
        self.cur = torch.zeros(B, n_cb, 1, dtype=torch.int64, device=self.dev)
        self.keys = np.zeros(B, dtype=np.int64)
        self.active = np.zeros(B, dtype=np.int64)
        m.set_active_streams(self.active)
        self.init = m._get_initial_token()[0].to(self.dev)
        self.pending = None   # the next request while it waits for rows or pages
        self.dirty = set()    # rows whose pages changed on the host since the last upload
        self.admitted = False
        # rows whose window can stop them run with the device's generation records (forward_step(gen_rows=True)):
        self.gen = False      # the last frame ran them
        self.fresh = set()    # rows admitted since the last frame (their records are uploaded before it)
        self.lagged = None    # (frame, slot, event, {row: state}, sums) of the last windowed frame, copied, not yet read
        self.status = None    # two pinned host slots for the statuses [B] int32, allocated on the first windowed frame
        self.status_slot = 0
        self.lp_frames: Dict[int, torch.Tensor] = {}   # best-of-N: windowed frame -> every row's sums after it (host)
        self.codec = codec
        if codec is not None:
            self.delay = _TTSDelay(m, B)
            self.card = codec.codebook_size
            cuda = self.dev.type == "cuda"
            self.pcm = [torch.zeros(B, codec.frame_size, dtype=torch.float32, pin_memory=cuda) for _ in range(2)]
            self.slot = 0
            self.in_flight = None         # (slot, event, chunk records) of the last frame run, not yet handed out

    def use_per_row(self) -> None:
        """from the next frame on, every row samples with its own settings (per-row tables)"""
        if self.default is None:
            self.default = self.imp.sampling()

    def occupied(self) -> List[int]:
        return [r for r in range(self.B) if self.rows[r] is not None]

    def _event(self):
        """a CUDA event recorded on the current stream after the work enqueued so far; None on a CPU device, where that
        work is done already"""
        if self.dev.type != "cuda":
            return None
        ev = torch.cuda.Event()
        ev.record()
        return ev

    def pages_needed(self, P: int, G: int) -> int:
        """KV pages of one request: its P + G positions, and with n_samples > 1 the N - 1 forked candidates' own pages
        (the prompt's full pages are shared)"""
        n = self.pages.pages_for(P + G)
        if self.n_samples > 1:
            n += self.pages.share_plan(P, P + G, self.n_samples - 1)[3]
        return n

    def fits(self, utt, P: int, G: int) -> None:
        """raise if the utterance needs more KV pages than the whole pool"""
        if self.paged and self.pages_needed(P, G) > self.pages.n_pages:
            raise RstnetError(f"utterance {utt!r} needs {self.pages_needed(P, G)} KV pages ({P + G} positions"
                              f"{f' x {self.n_samples} candidates' if self.n_samples > 1 else ''}), "
                              f"more than the whole pool of {self.pages.n_pages}")

    def admit(self, pull) -> None:
        """A request takes the n_samples lowest free rows once they and its pages are free; its prompt is prefilled into
        the first, and with n_samples > 1 forked into the others (their log-probability sums start from zero)."""
        m, pages, N = self.m, self.pages, self.n_samples
        groups = []   # (rows, request, prompt feed) admitted by this call
        taken = set()
        forked = 0    # pages the forks of this call's groups will take (they run after the prefill)
        while True:
            free = [r for r in range(self.B) if self.rows[r] is None and r not in taken]
            if len(free) < N:
                break
            if self.pending is None:
                req = pull()
                if req is None:
                    break
                self.fits(req.utt, req.P, req.G)
                self.pending = req
            req, rows = self.pending, free[:N]
            if self.paged:
                need = self.pages_needed(req.P, req.G)
                if need > pages.free - forked:
                    self.stats["wait_frames"] += 1
                    break
                forked += need - pages.pages_for(req.P + req.G)
                # it writes P positions in the prompt feed (init token + all prompt frames but the last) and one per
                # generated frame: at most P + G (G = maxlen; a row that stops runs one frame past its stop, at most
                # frame maxlen - 1)
                pages.reserve([rows[0]], req.P + req.G)
                self.dirty.add(rows[0])
            self.pending = None
            taken.update(rows)
            groups.append((rows, req, torch.cat([self.init, req.seq[:, :req.P].to(device=self.dev, dtype=torch.int64)], dim=1)))
        if self.dirty:
            # one upload of the table rows this frame's releases and admissions changed, before any launch
            m._state.upload_pages(sorted(self.dirty))
            self.dirty.clear()
        self.admitted = bool(groups)
        if not groups:
            return
        # the init token + all prompt frames but the last only feed the KV rings; the step on the last prompt frame
        # yields generated frame 0 (as generate)
        admitted = sorted(taken)
        m.reset_streaming(streams=admitted)
        if self.codec is not None:
            self.delay.reset(admitted)
            self.codec.reset_streaming(streams=admitted)
        if N > 1:
            if m._state.lp_acc is None:
                m._state.logprob_reset()
            m._state.logprob_reset(admitted)
        m.prefill_streams({rows[0]: feed[:, :-1] for rows, _, feed in groups})
        for rows, req, feed in groups:
            if N > 1:
                m.fork_kv(rows[0], rows[1:], req.P + req.G)
            for i, r in enumerate(rows):
                self.rows[r] = _Row(req.utt, req.P, req.G, self.n, req.sampling, req.task, req.minlen, req.windowed,
                                    cand=i, group=self.groups,
                                    forced=None if self.forced is None else self.forced.get(req.utt))
                self.keys[r] = sample_seed(req.seed, i)
                self.fresh.add(r)
                self.cur[r, :, 0] = feed[:, -1]
            self.groups += 1

    def _argmax(self, st: _Row) -> bool:
        """the row's audio heads take the argmax (no candidate masks: the whole card)"""
        sp = st.sampling if st.sampling is not None else (self.default or self.imp.sampling())
        return sp.heads()[1][0] == 0

    def _upload_records(self, rows: List[int]) -> None:
        """the generation records and next-frame candidate counts of these occupied rows, from the host's state"""
        recs, valid = [], []
        for r in rows:
            st = self.rows[r]
            argmax = self._argmax(st)
            kind = _lib.GEN_WINDOWED if st.windowed else _lib.GEN_FIXED
            recs.append([st.P, st.minlen, st.G, st.g, kind | (_lib.GEN_ARGMAX if argmax else 0)])
            valid.append([self.m.config.audio_card] * self.dep_q if argmax else
                         candidate_counts(st.P, st.minlen, st.g, self.dep_q))
        self.m._state.gen_rows_set(rows, recs, valid)

    def frame(self, records: Optional[list] = None) -> List[Tuple]:
        """One generated frame of every row (there must be an occupied row).  records: a list that receives a chunk
        record (row, row state, frame, chunk index, has PCM) of every row the frame ran, when the codec runs.  -> the
        rows finished: (utt, codes or None, raw frames [G', 9], row state)."""
        imp, m, B, rows = self.imp, self.m, self.B, self.rows
        occupied = self.occupied()
        mask = np.array([1 if rows[r] is not None else 0 for r in range(B)], dtype=np.int64)
        if not np.array_equal(mask, self.active):
            self.active = mask
            m.set_active_streams(self.active)
        gen = any(rows[r].windowed for r in occupied)
        table = None
        if gen:
            # a row whose window can stop it is in the batch: the device keeps every row's window and candidate counts
            fresh = occupied if not self.gen else sorted(self.fresh)
            if fresh:
                self._upload_records(fresh)
        else:
            table = torch.full((B, self.dep_q), 2048, dtype=torch.int32)
            for r in occupied:
                st = rows[r]
                table[r] = torch.tensor(candidate_counts(st.P, st.minlen, st.g, self.dep_q), dtype=torch.int32)
        self.gen = gen
        self.fresh.clear()
        per_row = None
        if self.default is not None:
            default = self.default
            per_row = [default if rows[r] is None or rows[r].sampling is None else rows[r].sampling for r in range(B)]
        extra = {"gen_rows": True} if gen else {}
        if self.n_samples > 1:
            extra["logprob"] = True
        if self.forced is not None:
            force = np.full((B, self.dep_q + 1), -1, dtype=np.int32)
            for r in occupied:
                if rows[r].forced is not None:
                    force[r] = rows[r].forced[:, rows[r].g]
            extra["force"] = torch.from_numpy(force).pin_memory() if self.dev.type == "cuda" else torch.from_numpy(force)
        toks = m.forward_step(self.cur, use_sampling=imp.use_sampling, temp_text=imp.temp_text, top_k_text=imp.top_k_text,
                              temp=imp.temp, top_k=imp.top_k, audio_valid=table,
                              sample_key=self.keys if self.admitted else None, depth_ring_quirk=False,
                              top_p_text=imp.top_p_text, top_p=imp.top_p, sampling=per_row, **extra)
        lagged = None
        if gen:
            # the frame's statuses: one copy to pinned host memory behind an event, read after the next frame is enqueued
            if self.status is None:
                cuda = self.dev.type == "cuda"
                self.status = [torch.zeros(B, dtype=torch.int32, pin_memory=cuda) for _ in range(2)]
            slot, self.status_slot = self.status_slot, self.status_slot ^ 1
            self.status[slot].copy_(m._state.gen_status[:B], non_blocking=True)
            lp = _to_host(m._state.logprob_sums()) if self.n_samples > 1 else None
            lagged = (self.n, slot, self._event(), {r: rows[r] for r in occupied if rows[r].windowed}, lp)
        if self.codec is not None:
            self._decode(toks)
        self.history[self.n] = toks
        self.n += 1
        self.stats["frames"] += 1
        self.stats["row_frames"] += len(occupied)
        self.cur = toks[:, :, None].clone()
        # the statuses of the frame before this one: the device has this frame queued while the host waits for them
        done = self.settle(keep_open=True)
        self.lagged = lagged
        lp = {}
        if self.n_samples > 1:
            last = [r for r in occupied if rows[r] is not None and not rows[r].windowed and rows[r].g + 1 == rows[r].G]
            if last:
                # the log-probability sums of the fixed rows this frame finishes: one copy to pinned host memory, not
                # waited for here (generate_many reads it after the next frame is enqueued)
                host, ev = _to_host(m._state.logprob_sums()[last]), self._event()
                lp = {r: (host, i, ev) for i, r in enumerate(last)}
        for r in occupied:
            st = rows[r]
            if st is None or st.start >= self.n:
                continue   # released above (it stopped at the frame before), or admitted after this frame
            st.g += 1
            if st.g == st.G:
                self._release(r)
                # a windowed row's status of this frame (kept, or stopped and dropped) is read with the next frame's
                if not st.windowed:
                    done.append(self._finish(st, r, self.n, False, lp.get(r)))
            if records is not None:
                # step g - 1 >= 1 completes codec frame g - 2; an utterance of one frame has no audio
                records.append((r, st, self.n - 1, max(st.g - 2, 0), st.g >= 2))
        freed = [r for r in occupied if rows[r] is None]
        if records is not None and freed:
            self.delay.reset(freed)   # a free row has no frame: the codec holds it
        self._prune()
        return done

    def _release(self, r: int) -> None:
        """free row r: park it at position 0 without pages (uploaded before the next launch)"""
        self.rows[r] = None
        self.m.reset_streaming(streams=[r])
        if self.paged:
            self.pages.release([r])
            self.dirty.add(r)

    def _finish(self, st: _Row, r: int, end: int, stopped: bool, lp: Optional[tuple]) -> Tuple:
        """Record the outcome of row r: frames st.start .. end - 1 kept (stopped: its stop rule fired on frame `end`), lp
        its log-probability sums.  -> (utt, codes [8, G' - 1] for the audio tasks else None, raw frames [G', 9], st)"""
        if end > st.start:
            raw = torch.stack([self.history[f][r] for f in range(st.start, end)])
        else:
            raw = torch.zeros(0, self.dep_q + 1, dtype=torch.int64, device=self.dev)
        st.end, st.stopped, st.lp = end, stopped, lp
        st.codes = reverse_delay(raw[:, 1:]) if st.task in AUDIO_TASKS else None
        if stopped:
            st.dropped = self.history[end][r]
        return st.utt, st.codes, raw, st

    def _prune(self) -> None:
        """drop the frames no running or unfinished row needs (a windowed row that ran its last frame is finished once
        that frame's statuses are read)"""
        live = [st for st in self.rows if st is not None]
        if self.lagged is not None:
            live += [st for st in self.lagged[3].values() if st.end is None]
        first = min([st.start for st in live], default=self.n)
        for f in [f for f in self.history if f < first]:
            del self.history[f]

    def settle(self, keep_open: bool = False) -> List[Tuple]:
        """Read the statuses of the last windowed frame (waits for its copy) and finish the rows they end: a row that
        stopped there (the frame and the one it ran after are dropped; it is released) and the rows that ran their last
        frame there.  keep_open: called from frame(), whose own statuses are still being copied."""
        lagged, self.lagged = self.lagged, None
        done = []
        if lagged is None:
            return done
        f, slot, ev, snap, lp = lagged
        if ev is not None:
            ev.synchronize()
        status = self.status[slot].numpy()
        if lp is not None:
            # best-of-N: each windowed frame's sums, kept while a row that ran it may still end there
            self.lp_frames = {k: v for k, v in self.lp_frames.items() if k >= f - 1}
            self.lp_frames[f] = lp
        for r, st in snap.items():
            stopped = int(status[r]) == _lib.GEN_STOPPED
            if self.rows[r] is st:
                if not stopped:
                    continue
                self._release(r)
            elif st.end is not None:
                continue   # it stopped at the frame before
            end = f if stopped else f + 1
            # the sums after frame end - 1: this frame's copy if it is kept, else the one before (or none)
            done.append(self._finish(st, r, end, stopped, None if lp is None else self._lp_at(end - 1, st, r)))
        if not keep_open:
            self._prune()
        return done

    def _lp_at(self, frame: int, st: _Row, r: int):
        """(host sums, row, event) of row r's log-probability sums after `frame` (zeros before its first frame); the
        copies were read by settle(), so no event is left to wait for"""
        if frame < st.start:
            return (torch.zeros(1, self.dep_q + 1, dtype=torch.float64), 0, None)
        return (self.lp_frames[frame], r, None)

    def _decode(self, toks: torch.Tensor) -> None:
        """the codec frame of every row that has one, into PCM slot self.slot"""
        out, valid = self.delay.step(toks)
        self.codec.set_active_streams(valid)
        pcm = self.codec.decode(out[:, 1:, None].clamp(max=self.card - 1))   # [B, 1, 1920]
        self.pcm[self.slot].copy_(pcm[:, 0], non_blocking=True)

    def stream_step(self, pull) -> Optional[List[TTSChunk]]:
        """Admit, run one frame with its codec step if a row is occupied, then hand out the previous frame's chunks.
        -> the chunks, or None when no row is occupied and nothing is left to hand out (nothing was launched)."""
        self.admit(pull)
        prev, self.in_flight = self.in_flight, None
        if self.occupied():
            records = []
            for _, _, _, st in self.frame(records):
                if not st.windowed:
                    st.codes = _to_host(st.codes)   # copied behind the slot's event; a windowed row's at hand-out
            self.in_flight, self.slot = (self.slot, self._event(), records), self.slot ^ 1
        elif prev is None:
            return None
        else:
            self.settle()   # the last frame's statuses, which decide its windowed rows' chunks
        return [] if prev is None else self._hand_out(*prev)

    def _hand_out(self, slot: int, ev, records) -> List[TTSChunk]:
        """The chunks of one frame's records, whose rows' outcomes are known by now (a windowed row's one frame late): a
        frame before the row's last kept one gives its PCM (a row's first frame has none), the last kept frame its chunk
        with the codes, and the frame a stop fired on (its chunk would decode the dropped frame) an empty chunk with the
        codes instead.  Nothing comes of the frame a row ran after its stop."""
        if ev is not None:
            ev.synchronize()
        pcm = self.pcm[slot].numpy()
        empty = torch.zeros(0, dtype=torch.float32)
        out = []
        for r, st, f, i, has_pcm in records:
            if st.end is None or f < st.end - 1:
                if has_pcm:
                    out.append(TTSChunk(st.utt, i, torch.from_numpy(pcm[r].copy()), None))
            elif f == st.end - 1:
                out.append(TTSChunk(st.utt, i, torch.from_numpy(pcm[r].copy()) if has_pcm else empty, st.codes.cpu()))
            elif f == st.end:
                out.append(TTSChunk(st.utt, i, empty, st.codes.cpu()))
        return out


def _ranked(cands, rank: Optional[str]) -> List[Candidate]:
    """[(finished row state, codes)] of one utterance -> its Candidates ranked; waits for the copy of their sums"""
    out = []
    for st, codes in cands:
        host, i, ev = st.lp
        if ev is not None:
            ev.synchronize()
        lp = host[i]
        out.append(Candidate(st.cand, codes, float(lp[1:].sum()), float(lp[0]), st.frames))
    return rank_candidates(out, rank)


def _to_host(t: torch.Tensor) -> torch.Tensor:
    """a host copy with t's strides, enqueued without waiting (pinned memory; valid once the stream has passed it)"""
    if t.device.type != "cuda":
        return t
    return torch.empty_like(t, device="cpu", pin_memory=True).copy_(t, non_blocking=True)


class _TTSDelay:
    """The TTS acoustic delay undone on the device by the Moshi delay-cache kernel (rstnet_lm_delay_cache_out): K = 9
    codebooks (text + 8 audio), delays [0, 0, 1, ..., 1], max_delay 1, ring of CT = 3 columns per (row, codebook).  After
    generated frame f of a row, out[row, 1:] is its codec frame f - 1 and valid[row] = 1 (f >= 1).  Rows held by the LM
    scope (its device `active` flags) keep their ring, step count and valid flag."""

    def __init__(self, m, B: int):
        dev, K = m.device, m.num_codebooks
        self.B, self.K, self.dep_q = B, K, K - 1
        self.delays = torch.tensor([0, 0] + [1] * (K - 2), dtype=torch.int64, device=dev)
        self.cache = torch.zeros(B, K, 3, dtype=torch.int64, device=dev)
        self.off = torch.zeros(B, dtype=torch.int64, device=dev)
        self.valid = torch.zeros(B, dtype=torch.int64, device=dev)
        self.out = torch.zeros(B, K, dtype=torch.int64, device=dev)
        self.lm_active = m._state.active

    def reset(self, rows) -> None:
        """the rows' step counts and valid flags back to 0"""
        idx = torch.as_tensor(rows, dtype=torch.int64).to(self.off.device)
        self.off[idx] = 0
        self.valid[idx] = 0

    def step(self, toks: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """toks: the frame's tokens [B, 9] (int64, rows contiguous) -> (out [B, 9], valid [B]), device buffers"""
        from . import _lib, ops
        if toks.dtype != torch.int64 or tuple(toks.shape) != (self.B, self.K) or toks.stride(1) != 1:
            raise RstnetError(f"the TTS delay takes int64 tokens [{self.B}, {self.K}] with contiguous rows")
        _lib.check(_lib.lib().rstnet_lm_delay_cache_out(
            self.cache.data_ptr(), self.off.data_ptr(), self.lm_active.data_ptr(), self.delays.data_ptr(), toks.data_ptr(),
            toks.stride(0), self.out.data_ptr(), self.K, self.valid.data_ptr(), self.B, self.K, self.dep_q, 3, 1,
            ops._stream()), "delay_cache_out")
        return self.out, self.valid
