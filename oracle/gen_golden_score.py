"""Generate tests/golden/lm_score.npz by running the UNMODIFIED reference's teacher-forced scoring here.

Run:  python -m oracle.gen_golden_score      (needs a checkout of the reference repository at REF)

The reference `models.llama_streaming.GPT` (small GQA / partial-rotary config of oracle/gen_golden_lm.gen_variant, seeded
synthetic weights) runs `GPT.forward` and `models.model.CrossEntropyAndAccuracy` on two sequences with pad frames,
fractional masks, ignore ids as labels and (second sequence) one codebook whose mask is zero throughout, in fp32 and bf16;
`InferenceImp.__call__` in mode 'teacher-force' is compiled from the reference file into its own namespace holding the
reference's CrossEntropyAndAccuracy.  oracle/score_oracle.py must reproduce the reference: the cross-entropy and the
temporal transformer bit for bit; the depth transformer to rounding, as gen_golden_lm documents for forward_local.
"""
from __future__ import annotations

import ast
import dataclasses
import os
import sys

os.environ.setdefault("NO_TORCH_COMPILE", "1")
os.environ.setdefault("NO_CUDA_GRAPH", "1")
sys.dont_write_bytecode = True

import numpy as np
import torch

from . import lm_oracle as L
from . import score_oracle as S
from .gen_golden import weights_digest
from .gen_golden_lm import GOLDEN, REF, reference_gpt, shrink

SEED = 17


def score_cfg():
    return dataclasses.replace(L.SMALL, n_query_groups=2, rotary_percentage=0.5,
                               rope_adjustments={"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                                 "original_max_seq_len": 32})


def score_inputs():
    """Two [9, 14] sequences with their masks: the last frames are pad frames (2049 / 128003, mask 0); masks hold 0, 0.5
    and 1; some real frames carry the ignore ids as labels; sequence 1 has codebook 5 masked out entirely (NaN loss)."""
    g = torch.Generator().manual_seed(23)
    seqs, masks = [], []
    for i, (L_, pad) in enumerate(((14, 3), (14, 5))):
        seq = torch.randint(0, 2048, (9, L_), generator=g)
        seq[0] = torch.randint(0, 150000, (L_,), generator=g)
        seq[1:, L_ - pad:] = S.AUDIO_PAD
        seq[0, L_ - pad:] = S.TEXT_PAD
        seq[2, 1], seq[7, 4], seq[0, 3] = S.AUDIO_PAD, S.AUDIO_PAD, S.TEXT_PAD
        mask = torch.ones(9, L_)
        mask[:, L_ - pad:] = 0.0
        pick = torch.rand(9, L_ - pad, generator=g)
        mask[:, :L_ - pad][pick < 0.25] = 0.5
        mask[:, :L_ - pad][pick > 0.85] = 0.0
        if i == 1:
            mask[1 + 5] = 0.0
        seqs.append(seq)
        masks.append(mask)
    return seqs, masks


def load_reference_teacher_force():
    """InferenceImp from infer_no_streaming.py (unmodified source, compiled alone as gen_golden_lm does) in a namespace
    that also holds the reference's CrossEntropyAndAccuracy, which its teacher-force branch calls."""
    sys.path.insert(0, REF)
    from models.model import CrossEntropyAndAccuracy
    from utils.sampling import sample_token, sample_token_audio, sample_token_audio_2048
    path = os.path.join(REF, "infer_no_streaming.py")
    tree = ast.parse(open(path).read())
    keep = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "InferenceImp"]
    assert len(keep) == 1
    ns = {"torch": torch, "CrossEntropyAndAccuracy": CrossEntropyAndAccuracy, "sample_token": sample_token,
          "sample_token_audio": sample_token_audio, "sample_token_audio_2048": sample_token_audio_2048}
    exec(compile(ast.Module(body=keep, type_ignores=[]), path, "exec"), ns)
    return ns["InferenceImp"], CrossEntropyAndAccuracy


def main():
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    cfg = score_cfg()
    RefImp, ref_ce = load_reference_teacher_force()
    seqs, masks = score_inputs()
    save = {"seqs": torch.stack(seqs).numpy(), "masks": torch.stack(masks).numpy()}
    w = L.synthetic_weights(cfg, seed=SEED, dtype=torch.float32, std=0.05)
    save["weights_sha256"] = np.array(weights_digest(w))
    for dtype, tag in ((torch.float32, "f32"), (torch.bfloat16, "bf16")):
        m = reference_gpt(w, cfg, dtype)
        m.load_state_dict({k: v.float() for k, v in w.items()}, strict=True)
        m = m.to(dtype)
        wd = {k: v.to(dtype) for k, v in w.items()}
        imp = RefImp(None, m, "teacher-force", 0.7, 25, 0.8, 30, "TTS")
        for i, (seq, mask) in enumerate(zip(seqs, masks)):
            with torch.no_grad():
                r_audio, r_text = m(seq.unsqueeze(0))
                r_la, r_lt = imp(seq.clone(), mask.clone())
                o = S.teacher_force(wd, cfg, seq, mask)
                s, mk = seq.unsqueeze(0), mask.unsqueeze(0)
                ra_loss, ra_m = ref_ce(r_audio, s[:, 1:], mk[:, 1:], [1] * 8, [S.AUDIO_PAD] * 8)
                rt_loss, rt_m = ref_ce(r_text.unsqueeze(2), s[:, 0].unsqueeze(1), mk[:, 0:1], [1], [S.TEXT_PAD])
                # the oracle's cross-entropy on the reference's own logits: bit for bit
                oa_loss, oa_m = S.cross_entropy_and_accuracy(r_audio, s[:, 1:], mk[:, 1:], [1] * 8, [S.AUDIO_PAD] * 8)
                ot_loss, ot_m = S.cross_entropy_and_accuracy(r_text.unsqueeze(2), s[:, 0].unsqueeze(1), mk[:, 0:1], [1], [S.TEXT_PAD])
            same = lambda a, b: torch.equal(a, b) or (bool(torch.isnan(a).all()) and bool(torch.isnan(b).all()))
            assert same(oa_loss, ra_loss) and same(ot_loss, rt_loss), (tag, i)
            for k in ("acc_all", "acc_target"):
                assert same(oa_m[k], ra_m[k]) and same(ot_m[k], rt_m[k]), (tag, i, k)
            assert same(r_la, ra_loss / 8) and same(r_lt, rt_loss), "InferenceImp teacher-force != its two calls"
            # the oracle's forward: temporal part (text logits) bit for bit, depth part to rounding
            assert torch.equal(o["text_logits"], r_text), (tag, i)
            d = (o["audio_logits"].float() - r_audio.float()).abs().max().item()
            assert d <= (2e-6 if dtype == torch.float32 else 4e-2) * max(1.0, r_audio.float().abs().max().item()), (tag, i, d)
            print(f"{tag} seq {i}: loss_audio/8 {float(r_la):.6f} loss_text {float(r_lt):.6f} acc_all {float(ra_m['acc_all']):.3f}; "
                  f"oracle cross-entropy == reference; forward_local max |diff| {d:.2e}")
            p = f"{tag}_{i}"
            save[f"{p}_loss_audio8"] = np.array(float(r_la), dtype=np.float64)
            save[f"{p}_loss_text"] = np.array(float(r_lt), dtype=np.float64)
            for k in ("acc_all", "acc_target"):
                save[f"{p}_audio_{k}"] = np.array(float(ra_m[k]), dtype=np.float64)
                save[f"{p}_text_{k}"] = np.array(float(rt_m[k]), dtype=np.float64)
            save[f"{p}_text_top"] = r_text[0].float().topk(8, dim=-1).values.numpy()
            save[f"{p}_text_argmax"] = r_text[0].float().argmax(-1).numpy()
            save[f"{p}_audio_argmax"] = r_audio[0].float().argmax(-1).numpy()
            if tag == "bf16":   # the GPU tests compare bf16 logits (a seeded sample of the columns, see shrink)
                save[f"{p}_audio_logits"] = r_audio[0].float().numpy()
    out = shrink(save)
    path = os.path.join(GOLDEN, "lm_score.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
