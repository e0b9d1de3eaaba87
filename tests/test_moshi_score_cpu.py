"""CPU tests of Moshi scoring: the oracle of the non-streaming forward against the reference's outputs
(tests/golden/moshi_score.npz), the pair-RoPE row-map entry point's declaration and argument checks, `score --model moshi`
parsing, the item checks and the pooled corpus summary."""
import math
import os

import numpy as np
import pytest
import torch

import moshi_score_oracle as O
from oracle import moshi_oracle as M
from oracle.gen_golden import weights_digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("tag,dtype", [("f32", torch.float32), ("bf16", torch.bfloat16)])
def test_moshi_score_oracle_matches_reference_golden(golden_dir, tag, dtype):
    g = np.load(os.path.join(golden_dir, "moshi_score.npz"))
    cfg = M.SMALL
    w = M.synthetic_weights(cfg, seed=5)
    assert weights_digest(w) == str(g["weights_sha256"])
    seqs, masks = O.score_inputs(cfg)
    assert np.array_equal(seqs.numpy(), g["seqs"]) and np.array_equal(masks.numpy(), g["masks"])
    assert seqs.shape[2] > cfg.context                       # the window slides
    wd = {k: v.to(dtype) for k, v in w.items()}
    with torch.no_grad():
        audio, text = O.forward(wd, cfg, seqs)
        met = O.validate(audio, text, seqs, masks)
    # the temporal transformer bit for bit
    tc = torch.from_numpy(g["text_cols"])
    assert torch.equal(text.float()[..., tc], torch.from_numpy(g[f"{tag}_text_logits"]))
    assert np.array_equal(text.float().argmax(-1).numpy(), g[f"{tag}_text_argmax"])
    # the depth transformer to rounding
    ac = torch.from_numpy(g["audio_cols"])
    ref = torch.from_numpy(g[f"{tag}_audio_logits"])
    d = float((audio.float()[..., ac] - ref).abs().max())
    assert d <= (2e-6 if dtype == torch.float32 else 4e-2) * max(1.0, float(ref.abs().max())), d
    for k in ("loss_audio", "loss_text", "acc_audio", "acc_text", "acc_target_audio", "acc_target_text"):
        r = float(g[f"{tag}_{k}"])
        assert abs(float(met[k]) - r) <= 1e-4 * max(1.0, abs(r)), (k, float(met[k]), r)


def test_rows_entry_point_declared_exported_and_checked():
    from rstnet_b200 import _lib
    name = "rstnet_lm_rope_pair_kv_append_rows_bf16"
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    assert f"int {name}(" in header and name in _lib.SYMBOLS
    lib = _lib.lib()
    fn = getattr(lib, name)
    assert fn.argtypes and len(fn.argtypes) == 13
    fake = 256                                                 # a pointer the checks never dereference
    good = [fake, fake, fake, fake, fake, fake, 5, 2, 4, 64, 200, fake, None]
    # (argument index, bad value, word expected in the error): every one returns before any launch
    for i, bad, word in ((0, None, b"null"), (1, None, b"null"), (2, None, b"row map"), (3, None, b"row map"),
                         (4, None, b"null"), (5, None, b"null"), (11, None, b"null"), (6, 0, b"shape"), (6, -3, b"shape"),
                         (7, 0, b"shape"), (8, 0, b"shape"), (9, 63, b"shape"), (9, 0, b"shape"), (10, 0, b"shape")):
        args = list(good)
        args[i] = bad
        assert fn(*args) != 0, (i, bad)
        assert word in lib.rstnet_last_error(), (i, lib.rstnet_last_error())


def test_score_cli_model_flag():
    from rstnet_b200.offline import build_parser
    base = ["score", "--input", "c.pt", "--config", "lm.json", "--checkpoint", "ck.pt", "--output-file", "o.json"]
    a = build_parser().parse_args(base + ["--model", "moshi", "--capacity", "4"])
    assert (a.model, a.config, a.checkpoint, a.capacity) == ("moshi", "lm.json", "ck.pt", 4)
    assert build_parser().parse_args(base).model == "gpt"
    with pytest.raises(SystemExit):
        build_parser().parse_args(base + ["--model", "llama"])


def test_moshi_score_item_checks():
    from rstnet_b200._lib import RstnetError
    from rstnet_b200.lm import score_item
    K = 17
    seq = torch.randint(0, 2048, (K, 5000))
    mask = torch.zeros(K, 5000)
    mask[:, :4000] = 1.0
    mask[12, 4500] = 0.5                                       # a user-stream codebook keeps frame 4500
    s, m, L = score_item(seq, mask, K)
    assert L == 4501 and s.shape == (K, 4501) and s.dtype == torch.int64 and m.dtype == torch.float32   # no length limit
    assert score_item(seq, torch.zeros(K, 5000), K)[2] == 0
    for bad in ((seq[:9], mask[:9]), (seq, mask[:, :10]), (seq[0], mask[0])):
        with pytest.raises(RstnetError):
            score_item(*bad, K)


def test_moshi_score_many_argument_checks():
    from rstnet_b200._lib import RstnetError
    from rstnet_b200.moshi import score_many

    class Fake:
        dep_q = 8
    with pytest.raises(RstnetError):
        next(score_many(Fake(), [], audio_weights=(1, 1)))
    with pytest.raises(RstnetError):
        next(score_many(Fake(), [], capacity=0))


def test_pooled_summary_is_token_weighted():
    from rstnet_b200.offline import moshi_score_summary
    aw = [100, 1, 1, 1, 1, 1, 1, 1]
    # utterance a: 2 tokens per codebook, b: 6 tokens per codebook; loss sums chosen so the per-utterance means differ
    a = {"frames": 2, "sums_audio": [[2.0, 2, 2, 1, 1]] * 8, "sums_text": [[4.0, 2, 1, 2, 1]]}
    b = {"frames": 6, "sums_audio": [[18.0, 6, 6, 3, 3]] * 8, "sums_text": [[6.0, 6, 6, 0, 0]]}
    s = moshi_score_summary({"a": a, "b": b}, aw)
    per_cb = (2.0 + 18.0) / (2 + 6)                            # 2.5 per token, not the mean of 1.0 and 3.0
    assert s["utterances"] == 2 and s["frames"] == 8
    assert s["loss_audio"] == pytest.approx(sum(aw) * per_cb, rel=1e-12)
    assert s["loss_text"] == pytest.approx(10.0 / 8, rel=1e-12)
    assert s["acc_audio"] == pytest.approx(4 / 8) and s["acc_target_audio"] == pytest.approx(4 / 8)
    assert s["acc_text"] == pytest.approx(2 / 8) and s["acc_target_text"] == pytest.approx(1 / 7)
    # a codebook masked out everywhere: NaN, as upstream
    c = {"frames": 1, "sums_audio": [[0.0, 0, 0, 0, 0]] * 8, "sums_text": [[1.0, 1, 1, 1, 1]]}
    assert math.isnan(moshi_score_summary({"c": c}, aw)["loss_audio"])
