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
    def __call__(self, seq: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        """seq [9, L] (one utterance, as upstream) -> codes [8, T'] after reverse_delay."""
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
            raise NotImplementedError("teacher-force mode is the training forward (out of scope)")

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
