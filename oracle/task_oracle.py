"""CPU oracle: the reference's generation loop `InferenceImp.__call__` for all four tasks (TTS, audio_only, text_only,
ASR), with its minlen / maxlen window and early stop.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): never imported by rstnet_b200/.

Reference: MLLM_v2/infer_no_streaming.py:184-308.  Per task (:184-226):
  * padding: text_only and ASR strip as many trailing frames as row 0 holds text pads (128003); audio_only and TTS as
    many as row 1 holds semantic pads (2049);
  * text_only / audio_only: the first L // 2 frames are the prompt, minlen = maxlen = L // 2;
  * TTS: the prompt is every frame but the text-empty ones (128002), minlen = maxlen = their count;
  * ASR: with e text-empty frames, the prompt is the first e + 1 frames, maxlen = L - e + 13, minlen = L - e - 13.
The loop (:229-292) samples codebook l > 0 from 2049 candidates once g_len = P + g_idx > minlen (all codebooks on the
first frame), and ends the utterance at the first codebook l > 2 whose token is >= 2048 while g_idx > minlen: that frame
is dropped.  The rule reads codebooks 3..7 only, never the semantic codebook 0; it is restated as written.

`lengths` = (minlen, maxlen) replaces the task's window (the reference has no such override); with (G, G) on TTS the
loop is oracle/infer_oracle.inference_imp_tts's, decision for decision.  Deterministic token rules only, as there.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

from . import lm_oracle as L
from .infer_oracle import ACOUSTIC_PAD, SEMANTIC_PAD, TEXT_EMPTY, TEXT_PAD, _deficit, _pick, reverse_delay

TASKS = ("TTS", "audio_only", "text_only", "ASR")


def layout(task: str, seq: torch.Tensor) -> Tuple[torch.Tensor, int, int, int]:
    """seq [9, L] -> (seq without its pad frames, prompt length P, minlen, maxlen) (infer_no_streaming.py:184-226)"""
    if task in ("text_only", "ASR"):
        pad_len = int(seq[0].eq(TEXT_PAD).int().sum().item())
    elif task in ("audio_only", "TTS"):
        pad_len = int(seq[1].eq(SEMANTIC_PAD).int().sum().item())
    else:
        raise NotImplementedError(task)
    seq = seq[:, :seq.shape[1] - pad_len]
    n = seq.shape[1]
    if task in ("text_only", "audio_only"):
        P = n // 2
        return seq, P, P, P
    empty = int(seq[0].eq(TEXT_EMPTY).int().sum().item())
    if task == "TTS":
        return seq, n - empty, empty, empty
    return seq, min(empty + 1, n), n - empty - 13, n - empty + 13   # prefix = seq[:, :, :empty + 1] (:219)


def n_valid(pre_gen_len: int, minlen: int, g_idx: int, l_idx: int) -> int:
    """candidate count of codebook l_idx at generated frame g_idx (infer_no_streaming.py:264-283)"""
    g_len = pre_gen_len + g_idx
    return 2049 if (g_len == pre_gen_len or (l_idx > 0 and g_len > minlen)) else 2048


def stops(g_idx: int, minlen: int, l_idx: int, token: int) -> bool:
    """the early stop (infer_no_streaming.py:284-286)"""
    return g_idx > minlen and l_idx > 2 and token >= 2048


def inference_imp(task: str, w: L.W, cfg: L.LMConfig, seq: torch.Tensor, use_sampling: bool,
                  lengths: Optional[Tuple[int, int]] = None, force: Optional[torch.Tensor] = None) -> Dict[str, object]:
    """InferenceImp.__call__ for `task`, n_samples == 1.  seq [9, L] int64.  Returns {"frames": [G', 9] the kept
    generated frames (text, audio 0..7), "margins": [G' + stopped, 9] (the stopped frame's row: its codebooks up to
    the one that stopped, +inf after), "stopped": bool, "P", "minlen", "maxlen", and for TTS "codes" [8, G' - 1]}.
    force [n, 9]: teacher-force these decisions for the first n frames (then the loop ends) and add "deficit" [n', 9] of
    the frames run (n' = G' + stopped; the stopped frame's row up to the codebook that stopped, 0 after)."""
    seq, P, minlen, maxlen = layout(task, seq)
    if lengths is not None:
        minlen, maxlen = int(lengths[0]), int(lengths[1])
    prefix = seq[:, :P].unsqueeze(0)
    init = torch.full((1, cfg.n_q + 1, 1), cfg.audio_card, dtype=torch.long)
    init[:, 0] = 151655
    pre_gen_len = P
    frames: List[torch.Tensor] = []
    margins: List[torch.Tensor] = []
    deficits: List[torch.Tensor] = []
    stopped = False
    n_frames = maxlen if force is None else min(maxlen, force.shape[0])
    for g_idx in range(n_frames):
        g_len = prefix.shape[2]
        global_prefix = torch.cat([init, prefix], dim=-1)
        transformer_out, text_logits = L.forward_global_full(w, cfg, global_prefix)
        prefix = torch.cat([prefix, torch.ones_like(prefix[:, :, 0:1]) * cfg.audio_card], dim=-1)
        text_tok, text_m = _pick(text_logits[:, -1:, :], use_sampling, text_logits.shape[-1])
        defs = []
        if force is not None:
            text_tok = force[g_idx, 0].reshape(1, 1)
            defs.append(_deficit(text_logits[:, -1:, :], text_tok, use_sampling, text_logits.shape[-1]))
        prefix[:, 0, -1] = text_tok.squeeze()
        toks, ms = [text_tok.reshape(())], [text_m.reshape(())]
        for l_idx in range(8):
            local_start = L.scaled_embedding(prefix[:, 0, :], w["codecformer_text_emb.weight"])
            logits = L.forward_local(w, cfg, local_start, prefix[:, 1:, :], transformer_out)
            valid = logits[:, -1:, l_idx:l_idx + 1, :]
            nv = n_valid(pre_gen_len, minlen, g_idx, l_idx)
            nxt, m = _pick(valid, use_sampling, nv)
            if force is not None:
                nxt = force[g_idx, l_idx + 1].reshape(1, 1, 1)
                defs.append(_deficit(valid, nxt, use_sampling, nv))
            ms.append(m.reshape(()))
            if stops(g_idx, minlen, l_idx, int(nxt)):
                stopped = True
                break
            prefix[:, l_idx + 1, g_len] = nxt.squeeze()
            toks.append(nxt.reshape(()))
        if stopped:
            margins.append(torch.cat([torch.stack(ms), torch.full((9 - len(ms),), float("inf"))]))
            if force is not None:
                deficits.append(torch.cat([torch.stack(defs), torch.zeros(9 - len(defs))]))
            break
        frames.append(torch.stack(toks))
        margins.append(torch.stack(ms))
        if force is not None:
            deficits.append(torch.stack(defs))
    fr = torch.stack(frames) if frames else torch.zeros(0, 9, dtype=torch.long)
    out = {"frames": fr, "margins": torch.stack(margins) if margins else torch.zeros(0, 9), "stopped": stopped,
           "P": P, "minlen": minlen, "maxlen": maxlen}
    if task == "TTS":
        out["codes"] = reverse_delay(fr[:, 1:]) if fr.shape[0] else torch.zeros(8, 0, dtype=torch.long)
    if force is not None:
        out["deficit"] = torch.stack(deficits) if deficits else torch.zeros(0, 9)
    return out


def reference_frames(final_results: torch.Tensor, prefix: torch.Tensor, pre_gen_len: int) -> torch.Tensor:
    """the reference loop's generated frames [G', 9] from its locals after the loop: the text row of `prefix` (written
    at infer_no_streaming.py:252) and the audio rows of `final_results` [G', 8]"""
    G = final_results.shape[0]
    return torch.cat([prefix[0, 0, pre_gen_len:pre_gen_len + G, None].cpu(), final_results.cpu()], dim=1)
