"""CPU oracle of the Moshi twin's non-streaming evaluation forward and of the reference trainer's validation metrics.

Test infrastructure only: never imported by rstnet_b200/.

Reference: MLLM_v2/models/model.py (LMModel.forward :297-319, forward_local :321-361, forward_text :364-389) over the
Kyutai StreamingTransformer outside a streaming scope (modules/transformer.py:375-419: positions 0..S-1, mask
(delta >= 0) & (delta < context), so the window slides once S > context), and validate_model
(MLLM/trainer/finetuning_full_fsdp.py:274-297: CrossEntropyAndAccuracy with audio weights [100, 1, ..., 1], ignore ids 2048 /
32000).  Pinned against the unmodified reference by scripts/gen_golden_moshi_score.py.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from oracle import lm_oracle as L
from oracle import moshi_oracle as M
from oracle.score_oracle import cross_entropy_and_accuracy

AUDIO_WEIGHTS = [100, 1, 1, 1, 1, 1, 1, 1]
IGNORE_AUDIO, IGNORE_TEXT = 2048, 32000


def forward_text(w: M.W, cfg: M.MoshiConfig, seq: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """LMModel.forward_text outside a streaming scope on seq [B, K, S] -> (transformer_out [B, S, dim], text_logits
    [B, 1, S, V])."""
    x = None
    for cb in range(cfg.n_q):
        e = L.scaled_embedding(seq[:, cb + 1], w[f"emb.{cb}.weight"])
        x = e if x is None else x + e
    x = x + L.scaled_embedding(seq[:, 0], w["text_emb.weight"])
    B, S, d = x.shape
    H = cfg.num_heads
    pos = torch.arange(S)
    delta = pos.view(-1, 1) - pos.view(1, -1)
    bias = (pos.view(1, -1) >= 0) & (delta >= 0) & (delta < cfg.context)
    for l in range(cfg.num_layers):
        p = f"transformer.layers.{l}"
        h = L.rms_norm_f32(x, w[f"{p}.norm1.alpha"])
        proj = F.linear(h, w[f"{p}.self_attn.in_proj_weight"])
        q, k, v = proj.view(B, S, 3, H, d // H).permute(2, 0, 3, 1, 4)
        q, k = M.rope_pairs(q, k, 0, cfg.max_period)
        a = F.scaled_dot_product_attention(q, k, v, bias, dropout_p=0.0).permute(0, 2, 1, 3).reshape(B, S, d)
        x = x + F.linear(a, w[f"{p}.self_attn.out_proj.weight"])
        h = L.rms_norm_f32(x, w[f"{p}.norm2.alpha"])
        g = F.linear(h, w[f"{p}.gating.linear_in.weight"]).view(B, S, 2, -1)
        x = x + F.linear(F.silu(g[..., 0, :]) * g[..., 1, :], w[f"{p}.gating.linear_out.weight"])
    out = L.rms_norm_f32(x, w["out_norm.alpha"])
    return out, F.linear(out, w["text_linear.weight"])[:, None]


def forward_local(w: M.W, cfg: M.MoshiConfig, local_start: torch.Tensor, sequence: torch.Tensor,
                  transformer_out: torch.Tensor) -> torch.Tensor:
    """LMModel.forward_local: the GPT oracle's teacher-forced depth transformer (the same module upstream) under the Moshi
    weight names.  -> logits [B, S, dep_q, card]."""
    depth = M.MoshiStream(w, cfg, 1).depth
    return L.forward_local(depth.w, depth.cfg, local_start, sequence, transformer_out)


def forward(w: M.W, cfg: M.MoshiConfig, seq: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """LMModel.forward (MLLM_v2): -> (audio_logits [B, S, dep_q, card], text_logits [B, S, V]).  The depth transformer
    starts from the text embedding of each INPUT frame and is fed the input frames' audio tokens."""
    B = seq.shape[0]
    start = torch.full((B, cfg.n_q + 1, 1), cfg.card, dtype=torch.long)
    start[:, 0] = cfg.text_card
    inputs = torch.cat([start, seq[:, :, :-1]], dim=2)
    out, text_logits = forward_text(w, cfg, inputs)
    local_start = L.scaled_embedding(inputs[:, 0, :], w["depformer_text_emb.weight"])
    return forward_local(w, cfg, local_start, inputs[:, 1:cfg.dep_q + 1, :], out), text_logits.squeeze(1)


def validate(audio_logits, text_logits, seqs, masks) -> Dict[str, torch.Tensor]:
    """validate_model's two CrossEntropyAndAccuracy calls on one batch."""
    la, ma = cross_entropy_and_accuracy(audio_logits, seqs[:, 1:9, :], masks[:, 1:9, :], AUDIO_WEIGHTS, [IGNORE_AUDIO] * 8)
    lt, mt = cross_entropy_and_accuracy(text_logits.unsqueeze(2), seqs[:, 0, :].unsqueeze(1), masks[:, 0:1, :], [1], [IGNORE_TEXT])
    return {"loss_audio": la, "loss_text": lt, "acc_audio": ma["acc_all"], "acc_text": mt["acc_all"],
            "acc_target_audio": ma["acc_target"], "acc_target_text": mt["acc_target"]}


def score_inputs(cfg: M.MoshiConfig, B: int = 2, S: int = 40, seed: int = 29):
    """B sequences [K, S] with their masks: masks of 0, 0.5 and 1, ignore ids used as labels, trailing all-zero-mask frames
    on sequence 1, and sequence 1's audio codebook 3 masked out entirely (NaN loss)."""
    g = torch.Generator().manual_seed(seed)
    K = cfg.n_q + 1
    seqs = torch.randint(0, cfg.card, (B, K, S), generator=g)
    seqs[:, 0] = torch.randint(0, cfg.text_card, (B, S), generator=g)
    pick = torch.rand(B, K, S, generator=g)
    seqs[:, 1:][pick[:, 1:] < 0.05] = IGNORE_AUDIO
    seqs[:, 0][pick[:, 0] < 0.05] = IGNORE_TEXT
    masks = torch.tensor([0.0, 0.5, 1.0, 1.0, 1.0])[torch.randint(0, 5, (B, K, S), generator=g)]
    masks[1, :, S - 4:] = 0.0
    masks[1, 1 + 3] = 0.0
    return seqs, masks
