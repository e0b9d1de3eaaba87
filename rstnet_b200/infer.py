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
Only the 'TTS' task is runnable upstream (the other branches reference undefined variables); same here.

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

from typing import Dict, Iterable, Iterator, List, Optional, Tuple

import numpy as np
import torch

from ._lib import RstnetError
from .lm import GPT, MAX_STREAMS


def candidate_counts(pre_gen_len: int, minlen: int, g_idx: int, dep_q: int = 8) -> List[int]:
    """Candidate-set size of each codebook at generated frame g_idx (infer_no_streaming.py:264-283): 2049 ids on the first
    generated frame and for codebooks > 0 once g_len > minlen, 2048 otherwise."""
    g_len = pre_gen_len + g_idx
    return [2049 if (g_len == pre_gen_len or (l > 0 and g_len > minlen)) else 2048 for l in range(dep_q)]


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
        self.semantic_pad_token = 2049
        self.text_empty_token = 128002
        self.mode = mode
        self.use_sampling = True          # upstream hard-codes True (:162); set the attribute to False for argmax decoding
        self.temp_text, self.top_k_text, self.temp, self.top_k = temp_text, top_k_text, temp, top_k

    @torch.no_grad()
    def __call__(self, seq: torch.Tensor, mask: torch.Tensor):
        """seq [9, L] (one utterance, as upstream) -> codes [8, T'] after reverse_delay.  In mode 'teacher-force'
        (infer_no_streaming.py:172-182, before any padding removal or task check) -> (loss_audio / 8, loss_text) as 0-dim
        fp64 tensors: score_many on this one utterance."""
        if self.mode == "teacher-force":
            _, met = next(self.score_many([(None, seq, mask)], capacity=1))
            return (torch.tensor(met["loss_audio"], dtype=torch.float64), torch.tensor(met["loss_text"], dtype=torch.float64))
        return self.generate(seq.unsqueeze(0).expand(self.n_samples, -1, -1))[0]

    @torch.no_grad()
    def generate(self, seq: torch.Tensor, return_frames: bool = False):
        """Batched form: seq [B, 9, L], all rows in the same TTS layout (same prompt length and number of frames to
        generate; row 0 defines them, as upstream reads `seq[0]`).  -> codes [B, 8, T'] (and the raw frames [B, G, 9])."""
        self._check_task()
        m = self.model
        dev = seq.device
        prefix_len, maxlen = self._layout(seq[0])
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
                                      temp=self.temp, top_k=self.top_k, audio_valid=valid, depth_ring_quirk=False)
                frames.append(toks)
                cur = toks[:, :, None]
            m.check_device_errors()
        raw = torch.stack(frames, dim=1).to(dev)                          # [B, G, 9]
        codes = torch.stack([reverse_delay(raw[b, :, 1:]) for b in range(B)], 0)
        return (codes, raw) if return_frames else codes

    def _check_task(self):
        if self.task_name != "TTS":
            raise NotImplementedError("only task 'TTS' is runnable in the reference loop (infer_no_streaming.py:184-226)")
        if self.mode == "teacher-force":
            raise NotImplementedError("teacher-force mode scores sequences (__call__ / score_many), it does not generate")

    def _score_item(self, seq, mask) -> Tuple[torch.Tensor, torch.Tensor, int]:
        """Host-side checks of one scoring item -> (seq int64 [9, L], mask fp32 [9, L], frames to score).  Trailing frames
        whose mask is zero in every codebook are dropped: the model is causal, so they change no earlier logit, and their
        rows add nothing to any sum."""
        m = self.model
        K = m.config.n_q + 1
        seq, mask = torch.as_tensor(seq), torch.as_tensor(mask)
        if seq.dim() != 2 or seq.shape[0] != K:
            raise RstnetError(f"a scored sequence is [{K}, L], got {tuple(seq.shape)}")
        if tuple(mask.shape) != tuple(seq.shape):
            raise RstnetError(f"the mask must have the sequence's shape {tuple(seq.shape)}, got {tuple(mask.shape)}")
        seq, mask = seq.to("cpu", torch.int64), mask.to("cpu", torch.float32)
        used = torch.nonzero((mask != 0).any(0))
        L = int(used[-1]) + 1 if used.numel() else 0
        if L > m.config.context:
            raise RstnetError(f"{L} frames to score (after dropping all-zero-mask frames) > context = {m.config.context}: "
                              "the non-streaming temporal transformer holds at most `context` positions")
        return seq[:, :L], mask[:, :L], L

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
        from .lm import cross_entropy_sums
        if not 1 <= capacity <= MAX_STREAMS:
            raise RstnetError(f"capacity must be in [1, {MAX_STREAMS}] (got {capacity})")
        m = self.model
        dev, c = m.device, m.config
        K, Q = m.num_codebooks, c.dep_q
        f32, i64 = torch.float32, torch.int64
        ign_text = torch.tensor([self.text_pad_token], dtype=i64, device=dev)
        ign_audio = torch.full((Q,), self.acoustic_pad_token, dtype=i64, device=dev)
        acc_text = torch.zeros(capacity, 1, 5, dtype=torch.float64, device=dev)
        acc_audio = torch.zeros(capacity, Q, 5, dtype=torch.float64, device=dev)
        source = iter(items)
        free, live, todo = list(range(capacity)), {}, []
        exhausted = False
        with m.streaming(capacity):
            st = m._state
            init = m._get_initial_token()[0]                                   # [9, 1]
            while True:
                admitted = []
                while free and not exhausted:
                    try:
                        utt, seq, mask = next(source)
                    except StopIteration:
                        exhausted = True
                        break
                    seq, mask, L = self._score_item(seq, mask)
                    if L == 0:
                        yield utt, self._score_metrics(torch.zeros(Q, 5, dtype=torch.float64), torch.zeros(1, 5, dtype=torch.float64), 0)
                        continue
                    s = free.pop(0)
                    feed = torch.cat([init, seq[:, :L - 1].to(dev)], dim=1)        # [initial token, seq[:, :-1]]
                    todo.append([s, feed.t().contiguous(), 0])
                    live[s] = dict(utt=utt, seq=seq.t().numpy(), mask=mask.t().numpy(), L=L)
                    admitted.append(s)
                if admitted:
                    m.reset_streaming(streams=admitted)
                    acc_text[admitted] = 0
                    acc_audio[admitted] = 0
                if not todo:
                    break
                ch, segs = st.row_chunk(todo, head=True)
                M = ch.M
                # labels / weights / accumulator slots of the chunk's rows; padding rows: ignore ids, weight 0, slot -1
                lab = np.empty((M, K), dtype=np.int64)
                lab[:, 0], lab[:, 1:] = self.text_pad_token, self.acoustic_pad_token
                w = np.zeros((M, K), dtype=np.float32)
                slot = np.full(M, -1, dtype=np.int32)
                for s, r0, t0, tn in segs:
                    u = live[s]
                    lab[r0:r0 + tn] = u["seq"][t0:t0 + tn]
                    w[r0:r0 + tn] = u["mask"][t0:t0 + tn]
                    slot[r0:r0 + tn] = s
                lab_d = torch.from_numpy(lab).to(dev)
                w_d = torch.from_numpy(w).to(dev)
                slot_d = torch.from_numpy(slot).to(dev)
                cross_entropy_sums(ch.logits, lab_d[:, 0].contiguous(), w_d[:, 0].contiguous(), 1, ign_text, slot_d, acc_text)
                dst = m._depth_state(M)
                if not hasattr(dst, "score_logits"):
                    dst.score_logits = torch.empty(M, Q, c.audio_card, dtype=torch.bfloat16, device=dev)
                dst.depth_teacher(ch.out, lab_d, dst.score_logits)
                cross_entropy_sums(dst.score_logits.view(M * Q, c.audio_card), lab_d[:, 1:].reshape(-1).contiguous(),
                                   w_d[:, 1:].reshape(-1).contiguous(), Q, ign_audio,
                                   slot_d.repeat_interleave(Q).contiguous(), acc_audio)
                done = [it for it in todo if it[2] == it[1].shape[0]]
                todo = [it for it in todo if it[2] < it[1].shape[0]]
                if done:
                    m.check_device_errors()
                    sa, stx = acc_audio.cpu(), acc_text.cpu()
                    for s, _, _ in done:
                        u = live.pop(s)
                        free.append(s)
                        yield u["utt"], self._score_metrics(sa[s], stx[s], u["L"])
            m.check_device_errors()

    def _layout(self, seq: torch.Tensor) -> Tuple[int, int]:
        """seq [9, L] -> (prompt length P, frames to generate G) after stripping the pad frames
        (infer_no_streaming.py:184-226)."""
        pad_len = int(seq[1].eq(self.semantic_pad_token).int().sum().item())
        L = seq.shape[1] - pad_len
        prefix_len = L - int(seq[0, :L].eq(self.text_empty_token).int().sum().item())
        if L - prefix_len <= 0:
            raise RstnetError("nothing to generate: the sequence has no text-empty frames")
        if prefix_len <= 0:
            raise RstnetError("the sequence has no prompt frames")
        return prefix_len, L - prefix_len

    @torch.no_grad()
    def generate_many(self, items: Iterable[Tuple[object, torch.Tensor]], capacity: int,
                      seeds: Optional[Dict[object, int]] = None, return_frames: bool = False) -> Iterator[Tuple]:
        """Continuous batching over (utt_id, seq [9, L]) items, each in its own TTS layout: yields (utt_id, codes [8, G-1])
        in completion order.  Up to `capacity` utterances decode together, one graph replay per frame; a finished row is
        held until the next utterance is admitted into it (its prompt fed through GPT.prefill_streams while the other
        rows keep their state).  Each utterance samples with its own candidate sets (candidate_counts) and its own random
        stream, keyed by seeds[utt_id] (default 0) and its own frame count from 0: with the defaults its codes are those
        of generate() on that utterance alone.  return_frames: yield (utt_id, codes, raw frames [G, 9]) as generate does."""
        self._check_task()
        if not 1 <= capacity <= MAX_STREAMS:
            raise RstnetError(f"capacity must be in [1, {MAX_STREAMS}] (got {capacity})")
        m, seeds = self.model, seeds or {}
        dev, B = m.device, capacity
        n_cb = m.num_codebooks
        dep_q = n_cb - 1                 # text + dep_q audio codebooks per frame
        source = iter(items)
        rows: List[Optional[dict]] = [None] * B
        history: Dict[int, torch.Tensor] = {}       # frame -> tokens [B, 9] of every row
        frame = 0
        cur = torch.zeros(B, n_cb, 1, dtype=torch.int64, device=dev)
        keys = np.zeros(B, dtype=np.int64)
        active = np.zeros(B, dtype=np.int64)
        with m.streaming(B):
            m.set_active_streams(active)
            init = m._get_initial_token()[0].to(dev)
            exhausted = False
            while True:
                admitted = {}
                for r in range(B):
                    if rows[r] is not None or exhausted:
                        continue
                    try:
                        utt, seq = next(source)
                    except StopIteration:
                        exhausted = True
                        break
                    P, G = self._layout(seq)
                    feed = torch.cat([init, seq[:, :P].to(device=dev, dtype=torch.int64)], dim=1)
                    admitted[r] = feed
                    rows[r] = dict(utt=utt, P=P, G=G, g=0, start=frame)
                    keys[r] = int(seeds.get(utt, 0))
                if admitted:
                    # the init token + all prompt frames but the last only feed the KV rings; the step on the last prompt
                    # frame yields generated frame 0 (as generate)
                    m.reset_streaming(streams=sorted(admitted))
                    m.prefill_streams({r: f[:, :-1] for r, f in admitted.items()})
                    for r, f in admitted.items():
                        cur[r, :, 0] = f[:, -1]
                occupied = [r for r in range(B) if rows[r] is not None]
                if not occupied:
                    break
                mask = np.array([1 if rows[r] is not None else 0 for r in range(B)], dtype=np.int64)
                if not np.array_equal(mask, active):
                    active = mask
                    m.set_active_streams(active)
                table = torch.full((B, dep_q), 2048, dtype=torch.int32)
                for r in occupied:
                    st = rows[r]
                    table[r] = torch.tensor(candidate_counts(st["P"], st["G"], st["g"], dep_q), dtype=torch.int32)
                toks = m.forward_step(cur, use_sampling=self.use_sampling, temp_text=self.temp_text, top_k_text=self.top_k_text,
                                      temp=self.temp, top_k=self.top_k, audio_valid=table,
                                      sample_key=keys if admitted else None, depth_ring_quirk=False)
                history[frame] = toks
                frame += 1
                cur = toks[:, :, None].clone()
                for r in occupied:
                    st = rows[r]
                    st["g"] += 1
                    if st["g"] == st["G"]:
                        raw = torch.stack([history[f][r] for f in range(st["start"], frame)])     # [G, 9]
                        rows[r] = None
                        m.reset_streaming(streams=[r])   # a held row keeps its position: park it at 0
                        codes = reverse_delay(raw[:, 1:])
                        yield (st["utt"], codes, raw) if return_frames else (st["utt"], codes)
                first = min([st["start"] for st in rows if st is not None], default=frame)
                for f in [f for f in history if f < first]:
                    del history[f]
            m.check_device_errors()
