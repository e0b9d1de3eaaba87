"""CPU checks of teacher-forced scoring: the oracle against the reference's outputs in tests/golden/lm_score.npz
(oracle/gen_golden_score.py), the `score` CLI's arguments and the host-side checks of InferenceImp.score_many."""
import os

import numpy as np
import pytest
import torch

from oracle import lm_oracle as L
from oracle import score_oracle as S
from oracle.gen_golden import weights_digest


def _score_cfg():
    import dataclasses
    return dataclasses.replace(L.SMALL, n_query_groups=2, rotary_percentage=0.5,
                               rope_adjustments={"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                                 "original_max_seq_len": 32})


def _close(a, b, rel):
    a, b = float(a), float(b)
    if np.isnan(b):
        return np.isnan(a)
    return abs(a - b) <= rel * max(1.0, abs(b))


@pytest.mark.parametrize("tag,dtype", [("f32", torch.float32), ("bf16", torch.bfloat16)])
def test_score_oracle_matches_reference_golden(golden_dir, tag, dtype):
    """The oracle's teacher-forced losses, accuracies and logits against the reference's.  The temporal transformer and
    the cross-entropy are bit-exact on the generating machine; the depth transformer's strided CPU GEMMs round by
    operand alignment (oracle/gen_golden_lm.py), so losses are compared to 1e-5 (fp32) / 2e-3 (bf16) and argmaxes may
    differ only where the top-2 margin is within that rounding."""
    g = np.load(os.path.join(golden_dir, "lm_score.npz"))
    cfg = _score_cfg()
    w = L.synthetic_weights(cfg, seed=17, dtype=torch.float32, std=0.05)
    assert weights_digest(w) == str(g["weights_sha256"])
    wd = {k: v.to(dtype) for k, v in w.items()}
    rel = 1e-5 if dtype == torch.float32 else 2e-3
    for i in range(g["seqs"].shape[0]):
        seq, mask = torch.from_numpy(g["seqs"][i]), torch.from_numpy(g["masks"][i])
        with torch.no_grad():
            o = S.teacher_force(wd, cfg, seq, mask)
        p = f"{tag}_{i}"
        assert _close(o["loss_audio"], g[f"{p}_loss_audio8"], rel), (p, float(o["loss_audio"]), float(g[f"{p}_loss_audio8"]))
        assert _close(o["loss_text"], g[f"{p}_loss_text"], rel)
        for k in ("acc_all", "acc_target"):
            assert _close(o["audio"][k], g[f"{p}_audio_{k}"], 0.0) and _close(o["text"][k], g[f"{p}_text_{k}"], 0.0)
        assert np.array_equal(o["text_logits"][0].float().argmax(-1).numpy(), g[f"{p}_text_argmax"])
        assert np.array_equal(o["text_logits"][0].float().topk(8, dim=-1).values.numpy(), g[f"{p}_text_top"])
        al = o["audio_logits"][0].float()
        top2 = al.topk(2, dim=-1).values
        tie = (top2[..., 0] - top2[..., 1]) <= 4 * rel * top2[..., 0].abs().clamp(min=1.0)
        agree = al.argmax(-1).numpy() == g[f"{p}_audio_argmax"]
        assert bool(np.all(agree | tie.numpy())), p
        if tag == "bf16":
            ref = torch.from_numpy(g[f"{p}_audio_logits"])
            mine = al[..., torch.from_numpy(g["logit_cols"])]
            assert float((mine - ref).abs().max()) <= 4e-2 * max(1.0, float(ref.abs().max()))
    # the NaN path: sequence 1 masks out codebook 5 entirely
    assert np.isnan(g["bf16_1_loss_audio8"]) and np.isfinite(g["bf16_0_loss_audio8"])


def test_exports_include_cross_entropy():
    from rstnet_b200 import _lib
    assert "rstnet_lm_cross_entropy_bf16" in _lib.SYMBOLS
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "rstnet_b200.h")).read()
    assert "int rstnet_lm_cross_entropy_bf16(" in header


def test_score_cli_arguments():
    from rstnet_b200.offline import build_parser
    a = build_parser().parse_args(["score", "--input", "c.pt", "--config", "cfg.json", "--checkpoint", "m.pt",
                                   "--output-file", "o.json", "--capacity", "3"])
    assert (a.cmd, a.input, a.config, a.checkpoint, a.output_file, a.capacity, a.device) == \
        ("score", "c.pt", "cfg.json", "m.pt", "o.json", 3, "cuda")
    assert build_parser().parse_args(["score", "--input", "c", "--config", "c", "--checkpoint", "c",
                                      "--output-file", "o"]).capacity == 8
    with pytest.raises(SystemExit):
        build_parser().parse_args(["score", "--input", "c.pt"])


def test_score_summary_is_the_reference_perplexity():
    from rstnet_b200.offline import score_summary
    m = {"a": {"loss_audio": 1.0, "loss_text": 3.0}, "b": {"loss_audio": 2.0, "loss_text": 5.0}}
    s = score_summary(m)
    assert s["utterances"] == 2 and s["loss_audio"] == 1.5 and s["loss_text"] == 4.0
    assert abs(s["perplexity_audio"] - float(np.exp(1.5))) < 1e-12


class _FakeModel:
    def __init__(self, context=16):
        from rstnet_b200.lm import Config
        self.config = Config(n_layer=1, n_embd=64, n_head=1, intermediate_size=64, n_q=8, dep_q=8, context=context)


def _imp(context=16):
    from rstnet_b200.infer import InferenceImp
    return InferenceImp(None, _FakeModel(context), "teacher-force", 0.7, 25, 0.8, 30, "TTS")


def test_score_item_host_checks():
    from rstnet_b200._lib import RstnetError
    imp = _imp(context=16)
    seq = torch.randint(0, 2048, (9, 20))
    mask = torch.zeros(9, 20)
    mask[:, :12] = 1.0
    mask[3, 14] = 0.5                       # last frame with a non-zero mask in some codebook: 14
    s, m, L = imp._score_item(seq, mask)
    assert L == 15 and s.shape == (9, 15) and m.shape == (9, 15) and s.dtype == torch.int64 and m.dtype == torch.float32
    assert torch.equal(s, seq[:, :15])
    assert imp._score_item(seq, torch.zeros(9, 20))[2] == 0
    with pytest.raises(RstnetError):
        imp._score_item(seq[:8], mask[:8])                      # not 9 codebooks
    with pytest.raises(RstnetError):
        imp._score_item(seq, mask[:, :19])                      # mask shape mismatch
    with pytest.raises(RstnetError):
        imp._score_item(seq[0], mask[0])                        # not [9, L]
    mask[:, 16] = 1.0
    with pytest.raises(RstnetError):
        imp._score_item(seq, mask)                              # 17 frames after trimming > context 16


def test_combine_sums_matches_the_reference_formula():
    from rstnet_b200.lm import combine_sums
    sums = torch.tensor([[3.0, 2, 1, 1, 1], [0.0, 0, 0, 0, 0], [5.0, 4, 4, 2, 2]], dtype=torch.float64)
    m = combine_sums(sums, [1, 1, 2])
    assert torch.isnan(m["loss"])                               # a group without a non-zero mask: 0/0 kept
    m = combine_sums(sums[[0, 2]], [1, 2])
    assert float(m["loss"]) == 3.0 / 2 + 2 * 5.0 / 4
    assert float(m["acc_all"]) == 3 / 6 and float(m["acc_target"]) == 3 / 5
