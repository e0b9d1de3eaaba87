"""CPU oracle of teacher-forced scoring: GPT.forward and CrossEntropyAndAccuracy.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): never imported by rstnet_b200/.

Reference: MLLM_v2/models/llama_streaming.py:651-663 (GPT.forward), MLLM_v2/models/model.py:31-65
(CrossEntropyAndAccuracy), MLLM_v2/infer_no_streaming.py:172-182 (the teacher-force branch of InferenceImp).  Pinned
against the unmodified reference by oracle/gen_golden_score.py.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from . import lm_oracle as L

TEXT_INITIAL, TEXT_PAD, AUDIO_PAD = 151655, 128003, 2049


def forward_teacher(w: L.W, cfg: L.LMConfig, seq: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """GPT.forward(seq [B, 9, S]) -> (audio_logits [B, S, dep_q, card], text_logits [B, S, V]) in the weights' dtype."""
    B = seq.shape[0]
    start = torch.full((B, cfg.n_q + 1, 1), cfg.audio_card, dtype=torch.long)
    start[:, 0] = TEXT_INITIAL
    out, text_logits = L.forward_global_full(w, cfg, torch.cat([start, seq[:, :, :-1]], dim=2))
    text_logits = text_logits.squeeze(1)
    local_start = L.scaled_embedding(seq[:, 0, :], w["codecformer_text_emb.weight"])
    return L.forward_local(w, cfg, local_start, seq[:, 1:cfg.dep_q + 1, :], out), text_logits


def cross_entropy_and_accuracy(logits, y, masks, loss_weights, ignore_ids):
    """CrossEntropyAndAccuracy, op for op: per group F.cross_entropy(ignore_index, reduction='none') * mask (in the
    logits' dtype, promoted by the mask), argmax, the != 0 / == 1 counts, loss += sum / count * weight."""
    loss = 0
    n_all = n_target = acc_tk = acc_target = 0
    for idx, _ in enumerate(loss_weights):
        m = masks[:, idx, :].reshape(-1)
        lg = logits[:, :, idx, :].reshape(-1, logits.shape[-1]).contiguous()
        t = y[:, idx, :].reshape(-1).contiguous()
        l = F.cross_entropy(lg, t, ignore_index=ignore_ids[idx], reduction="none") * m
        pred = lg.argmax(1)
        na = m.ne(0.0).int().sum()
        nt = m.eq(1.0).int().sum()
        acc_tk = acc_tk + torch.logical_and(pred.eq(t), m.ne(0.0)).int().sum()
        acc_target = acc_target + torch.logical_and(pred.eq(t), m.eq(1.0)).int().sum()
        n_all = n_all + na
        n_target = n_target + nt
        loss = loss + (l.sum() / na) * loss_weights[idx]
    metrics = {"acc_all": acc_tk / n_all, "acc_target": acc_target / n_target, "loss": loss.clone().detach()}
    return loss, metrics


def teacher_force(w: L.W, cfg: L.LMConfig, seq: torch.Tensor, mask: torch.Tensor) -> Dict[str, torch.Tensor]:
    """InferenceImp.__call__ in mode 'teacher-force' on seq [9, L], mask [9, L]: (loss_audio / 8, loss_text) and the
    metrics of both calls."""
    s, mk = seq.unsqueeze(0), mask.unsqueeze(0)
    audio_logits, text_logits = forward_teacher(w, cfg, s)
    la, ma = cross_entropy_and_accuracy(audio_logits, s[:, 1:, :], mk[:, 1:, :], [1] * 8, [AUDIO_PAD] * 8)
    lt, mt = cross_entropy_and_accuracy(text_logits.unsqueeze(2), s[:, 0, :].unsqueeze(1), mk[:, 0:1, :], [1], [TEXT_PAD])
    return {"loss_audio": la / 8, "loss_text": lt, "audio": ma, "text": mt, "audio_logits": audio_logits, "text_logits": text_logits}


def cross_entropy_f64(logits, y, masks, loss_weights, ignore_ids):
    """CrossEntropyAndAccuracy evaluated in float64 on the same (bf16-valued) logits: the yardstick of the kernel."""
    return cross_entropy_and_accuracy(logits.double(), y, masks.double(), loss_weights, ignore_ids)
