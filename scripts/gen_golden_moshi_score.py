"""Write tests/golden/moshi_score.npz from the reference's own non-streaming LMModel.forward and CrossEntropyAndAccuracy
(a CPU box with the reference sources; needs no GPU):

    python scripts/gen_golden_moshi_score.py --reference <RSTnet checkout>/MLLM_v2

The unmodified `models.model.LMModel` (the SMALL config of oracle/moshi_oracle.py: context 16, seeded synthetic weights)
runs `forward(seqs, masks)` on B = 2 sequences of S = 40 frames, so the attention window slides, followed by
validate_model's two CrossEntropyAndAccuracy calls (MLLM/trainer/finetuning_full_fsdp.py:274-297), in fp32 and bf16.
tests/moshi_score_oracle.py must reproduce the reference: the temporal transformer (text logits) and the cross-entropy on
the reference's own logits bit for bit, the depth transformer to rounding (as oracle/gen_golden_lm.py documents for
forward_local).  The inputs have fractional masks, ignore ids used as labels, trailing all-zero-mask frames and one
audio codebook whose mask is zero throughout.  Logits are stored on a seeded sample of their columns.
"""
from __future__ import annotations

import argparse
import os
import sys

os.environ.setdefault("NO_TORCH_COMPILE", "1")
os.environ.setdefault("NO_CUDA_GRAPH", "1")
sys.dont_write_bytecode = True

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import moshi_score_oracle as O  # noqa: E402
from oracle import moshi_oracle as M  # noqa: E402
from oracle.gen_golden import weights_digest  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "moshi_score.npz")
SEED = 5
COLS = 64   # logit columns kept per row


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--reference", required=True, help="the reference's MLLM_v2 directory")
    args = ap.parse_args()
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    sys.path.insert(0, args.reference)
    from models.model import CrossEntropyAndAccuracy, LMModel
    cfg = M.SMALL
    seqs, masks = O.score_inputs(cfg)
    w = M.synthetic_weights(cfg, seed=SEED)
    rng = np.random.default_rng(0)
    text_cols = np.sort(rng.choice(cfg.text_card, COLS, replace=False))
    audio_cols = np.sort(rng.choice(cfg.card, COLS, replace=False))
    save = {"seqs": seqs.numpy(), "masks": masks.numpy(), "weights_sha256": np.array(weights_digest(w)),
            "text_cols": text_cols, "audio_cols": audio_cols}
    same = lambda a, b: torch.equal(a, b) or (bool(torch.isnan(a).all()) and bool(torch.isnan(b).all()))
    for dtype, tag in ((torch.float32, "f32"), (torch.bfloat16, "bf16")):
        m = LMModel(**cfg.reference_kwargs()).eval()
        assert set(m.state_dict().keys()) == set(w.keys()), set(m.state_dict().keys()) ^ set(w.keys())
        m.load_state_dict(w, strict=True)
        m = m.to(dtype)
        wd = {k: v.to(dtype) for k, v in w.items()}
        with torch.no_grad():
            r_audio, r_text = m(seqs, masks)
            la, ma = CrossEntropyAndAccuracy(r_audio, seqs[:, 1:9, :], masks[:, 1:9, :], loss_weights=O.AUDIO_WEIGHTS,
                                             ignore_ids=[O.IGNORE_AUDIO] * 8)
            lt, mt = CrossEntropyAndAccuracy(r_text.unsqueeze(2), seqs[:, 0, :].unsqueeze(1), masks[:, 0:1, :], loss_weights=[1],
                                             ignore_ids=[O.IGNORE_TEXT])
            mine = O.validate(r_audio, r_text, seqs, masks)
            o_audio, o_text = O.forward(wd, cfg, seqs)
        ref = {"loss_audio": la, "loss_text": lt, "acc_audio": ma["acc_all"], "acc_text": mt["acc_all"],
               "acc_target_audio": ma["acc_target"], "acc_target_text": mt["acc_target"]}
        for k, v in ref.items():
            assert same(mine[k], v), (tag, k, mine[k], v)                 # the oracle's metrics on the reference's logits
        assert torch.equal(o_text, r_text), f"oracle forward_text != reference ({tag})"
        d = (o_audio.float() - r_audio.float()).abs().max().item()
        assert d <= (2e-6 if dtype == torch.float32 else 4e-2) * max(1.0, r_audio.float().abs().max().item()), (tag, d)
        print(f"{tag}: loss_audio {float(la):.6f} loss_text {float(lt):.6f} acc_audio {float(ma['acc_all']):.4f}; oracle "
              f"forward_text and cross-entropy == reference; forward_local max |diff| {d:.2e}")
        for k, v in ref.items():
            save[f"{tag}_{k}"] = np.array(float(v), dtype=np.float64)
        save[f"{tag}_text_logits"] = r_text.float()[..., text_cols].numpy()
        save[f"{tag}_text_argmax"] = r_text.float().argmax(-1).numpy()
        save[f"{tag}_audio_logits"] = r_audio.float()[..., audio_cols].numpy()
        save[f"{tag}_audio_argmax"] = r_audio.float().argmax(-1).numpy()
    np.savez_compressed(OUT, **save)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
