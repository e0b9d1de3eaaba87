"""GPU tests of teacher-forced scoring (-m gpu): the cross-entropy kernel against a float64 evaluation of the same bf16
logits, CrossEntropyAndAccuracy against the reference's formula in float64, GPT.forward and teacher-force
InferenceImp.__call__ against the reference's outputs (tests/golden/lm_score.npz), and InferenceImp.score_many against
scoring each utterance alone."""
import dataclasses
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import lm_oracle as L
from oracle import score_oracle as S
from rstnet_b200 import _lib
from rstnet_b200.infer import InferenceImp
from rstnet_b200.lm import GPT, Config, CrossEntropyAndAccuracy, cross_entropy_sums

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16


def _product_config(cfg, **kw):
    return Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                  n_query_groups=cfg.n_kv, rotary_percentage=cfg.rotary_percentage, rope_adjustments=cfg.rope_adjustments,
                  intermediate_size=cfg.intermediate_size, norm_eps=cfg.norm_eps, padded_vocab_size=cfg.padded_vocab_size,
                  audio_card=cfg.audio_card, n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim,
                  codecformer_heads=cfg.codecformer_heads, codecformer_layers=cfg.codecformer_layers,
                  codecformer_dim_feedforward=cfg.codecformer_dim_feedforward, context=cfg.context, **kw)


def _score_cfg(**kw):
    return dataclasses.replace(L.SMALL, n_query_groups=2, rotary_percentage=0.5,
                               rope_adjustments={"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                                 "original_max_seq_len": 32}, **kw)


def _model(cfg, seed):
    w32 = L.synthetic_weights(cfg, seed=seed, dtype=torch.float32, std=0.05)
    m = GPT(_product_config(cfg))
    m.load_state_dict(w32, strict=True)
    return m.to(DEV, BF).eval(), {k: v.to(BF) for k, v in w32.items()}


@pytest.fixture(scope="module")
def gqa():
    return _model(_score_cfg(), 17) + (_score_cfg(),)


@pytest.fixture(scope="module")
def mha():
    return _model(L.SMALL, 7) + (L.SMALL,)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-6))


def _cos(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float(torch.dot(a, b) / (a.norm() * b.norm()).clamp(min=1e-12))


# ------------------------------------------------------------------------------------------------ the kernel
def _ce_case(V, stride, rows, groups, seed, offset=0):
    g = torch.Generator().manual_seed(seed)
    buf = (torch.randn(rows * stride + offset + 8, generator=g) * 3.0).to(BF).to(DEV)
    lg = buf[offset:offset + rows * stride].view(rows, stride)[:, :V]
    ign = torch.randint(0, V, (groups,), generator=g)
    y = torch.randint(0, V, (rows,), generator=g)
    pick = torch.rand(rows, generator=g)
    y[pick < 0.1] = ign[torch.arange(rows)[pick < 0.1] % groups]                       # ignore ids as labels
    lg_f = lg.float()
    am = lg_f.argmax(-1).cpu()
    y[(pick > 0.6) & (pick < 0.8)] = am[(pick > 0.6) & (pick < 0.8)]                   # correct predictions
    w = torch.tensor([0.0, 0.5, 1.0, 1.0, 0.25], dtype=torch.float32)[torch.randint(0, 5, (rows,), generator=g)]
    # planted: duplicate maxima (first index wins), a NaN logit (on an ignored row: loss 0, pred = the NaN's index)
    r0 = 0
    mx = float(lg_f[r0].max()) + 1.0
    lg[r0, V // 3] = mx
    lg[r0, (2 * V) // 3] = mx
    lg[r0, V - 1] = mx
    if rows > 1:
        lg[1, V // 2] = float("nan")
        lg[1, V // 2 + 1] = float("nan")
        y[1] = ign[1 % groups]
    return lg, y.to(DEV), w.to(DEV), ign.to(DEV)


def _ce_ref64(lg, y, ign, groups):
    x = lg.double()
    rows, V = x.shape
    lse = torch.logsumexp(x, -1)
    yi = y.clamp(0, V - 1)
    nll = lse - x.gather(1, yi[:, None])[:, 0]
    g = torch.arange(rows, device=x.device) % groups
    nll = torch.where(y == ign[g], torch.zeros_like(nll), nll)
    return nll, lg.argmax(-1)


@pytest.mark.parametrize("V,stride,rows,groups,offset", [
    (2050, 2051, 300, 8, 0), (2050, 2050, 1, 1, 0), (2050, 2051, 37, 1, 1), (1001, 1001, 300, 1, 0), (1001, 1003, 64, 8, 3),
    (152064, 152064, 33, 1, 0), (152064, 152067, 16, 8, 1), (152064, 152064, 1, 1, 0)])
def test_cross_entropy_kernel_vs_float64(V, stride, rows, groups, offset):
    lg, y, w, ign = _ce_case(V, stride, rows, groups, seed=V + rows + groups, offset=offset)
    acc, nll, pred = cross_entropy_sums(lg, y, w, groups, ign)
    torch.cuda.synchronize()
    ref, ref_pred = _ce_ref64(lg, y, ign, groups)
    assert torch.equal(pred.long(), ref_pred), "pred must be torch.argmax (first maximum, NaN as the maximum)"
    assert int(pred[0]) == V // 3
    if rows > 1:
        assert int(pred[1]) == V // 2 and float(nll[1]) == 0.0
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isfinite(nll.double()), fin)
    err = ((nll.double() - ref).abs() / ref.abs().clamp(min=1e-30))[fin & (ref != 0)]
    worst = float(err.max()) if err.numel() else 0.0
    assert worst <= 2e-6, worst
    ignored = y == ign[torch.arange(rows, device=DEV) % groups]
    assert bool((nll[ignored] == 0).all())
    # the accumulator: the float64 sums of the kernel's own rows
    g = torch.arange(rows, device=DEV) % groups
    ok = pred.long() == y
    for gi in range(groups):
        sel = g == gi
        want = [float((w[sel].double() * nll[sel].double()).sum()), int((w[sel] != 0).sum()), int((w[sel] == 1).sum()),
                int((ok & sel & (w != 0)).sum()), int((ok & sel & (w == 1)).sum())]
        got = acc[0, gi].tolist()
        assert got[1:] == want[1:], (gi, got, want)
        assert abs(got[0] - want[0]) <= 1e-12 * max(1.0, abs(want[0])), (gi, got[0], want[0])
        assert int((ignored & sel & (w != 0)).sum()) <= got[1]                        # ignored rows are still counted
    acc2, nll2, pred2 = cross_entropy_sums(lg, y, w, groups, ign)
    assert torch.equal(acc, acc2) and torch.equal(nll, nll2) and torch.equal(pred, pred2), "identical calls, identical bytes"


def test_cross_entropy_row_slots_and_padding():
    lg, y, w, ign = _ce_case(2050, 2051, 96, 8, seed=5)
    slot = torch.tensor([i // 8 % 3 if i < 80 else -1 for i in range(96)], dtype=torch.int32, device=DEV)
    acc = torch.zeros(3, 8, 5, dtype=torch.float64, device=DEV)
    _, nll, pred = cross_entropy_sums(lg, y, w, 8, ign, slot, acc)
    whole, _, _ = cross_entropy_sums(lg[:80], y[:80], w[:80], 8, ign)
    torch.cuda.synchronize()
    assert bool((pred[80:] == -1).all()) and bool((nll[80:] == 0).all())
    assert torch.equal(acc[:, :, 1:].sum(0), whole[0, :, 1:])
    assert torch.allclose(acc[:, :, 0].sum(0), whole[0, :, 0], rtol=1e-12, atol=0)
    for s in range(3):
        rows = [i for i in range(80) if i // 8 % 3 == s]
        one, _, _ = cross_entropy_sums(lg[rows], y[rows], w[rows], 8, ign)
        assert torch.equal(acc[s, :, 1:], one[0, :, 1:])


def test_out_of_range_label_poisons_row_and_raises(mha):
    m = mha[0]
    lg, y, w, ign = _ce_case(2050, 2051, 20, 1, seed=9)
    m.check_device_errors()                     # clean start
    y[3], y[7] = 2050, -5
    _, nll, _ = cross_entropy_sums(lg, y, w, 1, ign)
    assert torch.isnan(nll[3]) and torch.isnan(nll[7]) and bool(torch.isfinite(nll[:3]).all())
    with pytest.raises(IndexError):
        m.check_device_errors()
    m.check_device_errors()                     # cleared
    B, T = 1, 6
    with pytest.raises(IndexError):
        CrossEntropyAndAccuracy(lg[:T].reshape(B, T, 1, 2050), torch.full((B, 1, T), 4000, device=DEV),
                                torch.ones(B, 1, T, device=DEV), [1], [2049])


def test_cross_entropy_kernel_is_graph_capturable():
    lg, y, w, ign = _ce_case(2050, 2051, 64, 8, seed=11)
    acc = torch.zeros(1, 8, 5, dtype=torch.float64, device=DEV)
    nll = torch.empty(64, dtype=torch.float32, device=DEV)
    pred = torch.empty(64, dtype=torch.int32, device=DEV)
    eager, n0, p0 = cross_entropy_sums(lg, y, w, 8, ign)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            cross_entropy_sums(lg, y, w, 8, ign, acc=acc, nll=nll, pred=pred)
    acc.zero_()
    gr.replay()
    torch.cuda.synchronize()
    assert torch.equal(acc, eager) and torch.equal(nll, n0) and torch.equal(pred, p0)


# --------------------------------------------------------------------------------- CrossEntropyAndAccuracy
@pytest.mark.parametrize("B,T,G,V,nan_group", [(2, 37, 8, 2050, None), (2, 37, 8, 2050, 5), (1, 23, 1, 152064, None)])
def test_cross_entropy_and_accuracy_vs_reference_formula_f64(B, T, G, V, nan_group):
    g = torch.Generator().manual_seed(B * T + G)
    logits = (torch.randn(B, T, G, V, generator=g) * 2).to(BF)
    y = torch.randint(0, min(V, 2048), (B, G, T), generator=g)
    am = logits.float().argmax(-1).permute(0, 2, 1)
    pick = torch.rand(B, G, T, generator=g)
    y = torch.where(pick < 0.3, am, y)
    ign = [2049] * G if G > 1 else [128003]
    y[pick > 0.9] = ign[0]
    masks = torch.tensor([0.0, 0.5, 1.0, 1.0])[torch.randint(0, 4, (B, G, T), generator=g)]
    if nan_group is not None:
        masks[:, nan_group] = 0.0
    lw = [1] * G
    loss, met = CrossEntropyAndAccuracy(logits.to(DEV), y.to(DEV), masks.to(DEV), lw, ign)
    r_loss, r_met = S.cross_entropy_f64(logits, y, masks, lw, ign)
    if nan_group is not None:
        assert math.isnan(float(loss)) and math.isnan(float(r_loss))
    else:
        assert abs(float(loss) - float(r_loss)) <= 1e-6 * abs(float(r_loss)), (float(loss), float(r_loss))
    # exact counts: the reference's ratio of two int tensors is float32, ours fp64 (one count apart is >= 1/N)
    for k in ("acc_all", "acc_target"):
        assert abs(float(met[k]) - float(r_met[k])) <= 1e-6 * float(r_met[k]), (k, float(met[k]), float(r_met[k]))
    assert float(met["loss"]) == float(loss) or math.isnan(float(loss))


# ------------------------------------------------------------------------------------ GPT.forward, teacher force
def _forward_checks(m, wd, cfg, seq, gold=None, p=None):
    """our bf16 deviation from an fp32 evaluation of the same bf16 weights <= 2x the reference's (golden) or the bf16
    oracle's own deviation, cosine >= 0.999."""
    audio, text = m(seq[None].to(DEV))
    assert audio.shape == (1, seq.shape[1], cfg.dep_q, cfg.audio_card) and audio.dtype == BF
    assert text.shape == (1, seq.shape[1], cfg.padded_vocab_size) and text.dtype == BF
    with torch.no_grad():
        t_audio, t_text = S.forward_teacher({k: v.float() for k, v in wd.items()}, cfg, seq[None])
        b_audio, b_text = S.forward_teacher(wd, cfg, seq[None])
    if gold is not None:
        cols = torch.from_numpy(gold["logit_cols"])
        ref = torch.from_numpy(gold[f"{p}_audio_logits"])[None]
        mine, truth = audio.float().cpu()[..., cols], t_audio.float()[..., cols]
        assert _cos(mine, ref) >= 0.999
        assert _rel(mine, truth) <= 2.0 * _rel(ref, truth) + 1e-2, (_rel(mine, truth), _rel(ref, truth))
        top = text[0].float().topk(8, dim=-1).values.cpu()
        assert _rel(top, torch.from_numpy(gold[f"{p}_text_top"])) <= 8e-2
    for mine, bf, truth in ((audio, b_audio, t_audio), (text, b_text, t_text)):
        assert _cos(mine, bf) >= 0.999
        assert _rel(mine, truth) <= 2.0 * _rel(bf, truth) + 1e-2, (_rel(mine, truth), _rel(bf, truth))
    return audio, text


def test_gpt_forward_gqa_vs_reference_golden(golden_dir, gqa):
    m, wd, cfg = gqa
    gold = np.load(os.path.join(golden_dir, "lm_score.npz"))
    for i in range(gold["seqs"].shape[0]):
        _forward_checks(m, wd, cfg, torch.from_numpy(gold["seqs"][i]), gold, f"bf16_{i}")
    with m.streaming(1):
        with pytest.raises(_lib.RstnetError):
            m(torch.from_numpy(gold["seqs"][0])[None].to(DEV))
    with pytest.raises(_lib.RstnetError):
        m(torch.from_numpy(gold["seqs"][0])[None].to(DEV), input_pos=torch.arange(3))
    with pytest.raises(_lib.RstnetError):
        m(torch.zeros(1, 9, cfg.context + 1, dtype=torch.int64, device=DEV))


def test_gpt_forward_mha_vs_oracle(mha):
    m, wd, cfg = mha
    g = torch.Generator().manual_seed(41)
    seq = torch.randint(0, 2048, (9, 13), generator=g)
    seq[0] = torch.randint(0, 150000, (13,), generator=g)
    _forward_checks(m, wd, cfg, seq)


def test_teacher_force_call_vs_reference_golden(golden_dir, gqa):
    m, wd, cfg = gqa
    gold = np.load(os.path.join(golden_dir, "lm_score.npz"))
    imp = InferenceImp(None, m, "teacher-force", 0.7, 25, 0.8, 30, "whatever")   # any task name: checked after this branch
    w32 = {k: v.float() for k, v in wd.items()}
    for i in range(gold["seqs"].shape[0]):
        seq, mask = torch.from_numpy(gold["seqs"][i]), torch.from_numpy(gold["masks"][i])
        la, lt = imp(seq.to(DEV), mask.to(DEV))
        with torch.no_grad():
            truth = S.teacher_force(w32, cfg, seq, mask)
        for mine, key, t in ((la, "loss_audio8", truth["loss_audio"]), (lt, "loss_text", truth["loss_text"])):
            ref = float(gold[f"bf16_{i}_{key}"])
            if math.isnan(ref):
                assert math.isnan(float(mine)) and math.isnan(float(t))
                continue
            assert abs(float(mine) - float(t)) <= 2.0 * abs(ref - float(t)) + 1e-3 * abs(float(t)), (i, key, float(mine), ref, float(t))


# ------------------------------------------------------------------------------------------------ score_many
def _ragged_items(seed, lengths):
    g = torch.Generator().manual_seed(seed)
    items = []
    for j, Lj in enumerate(lengths):
        seq = torch.randint(0, 2048, (9, Lj), generator=g)
        seq[0] = torch.randint(0, 150000, (Lj,), generator=g)
        pick = torch.rand(9, Lj, generator=g)
        seq[1:][pick[1:] < 0.05] = 2049
        seq[0][pick[0] < 0.05] = 128003
        mask = torch.tensor([0.0, 0.5, 1.0, 1.0, 1.0])[torch.randint(0, 5, (9, Lj), generator=g)]
        items.append((f"u{j}", seq, mask))
    return items


@pytest.fixture(scope="module")
def long_ctx():
    cfg = _score_cfg(context=256, block_size=512)
    return _model(cfg, 17) + (cfg,)


def _alone(m, seq, mask):
    """CrossEntropyAndAccuracy(GPT.forward(seq)) on one utterance, with the per-group sums and bf16 tie counts."""
    audio, text = m(seq[None].to(DEV))
    text = text.view(1, seq.shape[1], -1)          # GPT.forward squeezes dim 1 as upstream: [1, V] for one frame
    s, mk = seq[None].to(DEV), mask[None].to(DEV)
    la, ma = CrossEntropyAndAccuracy(audio, s[:, 1:], mk[:, 1:], [1] * 8, [2049] * 8)
    lt, mt = CrossEntropyAndAccuracy(text.unsqueeze(2), s[:, 0].unsqueeze(1), mk[:, 0:1], [1], [128003])
    ties = []   # rows whose bf16 top-2 margin is within one bf16 step of the maximum: rounding may flip their argmax
    for lg in (audio.float().reshape(-1, audio.shape[-1]), text.float().reshape(-1, text.shape[-1])):
        t2 = lg.topk(2, dim=-1).values
        ties.append(int(((t2[:, 0] - t2[:, 1]) <= t2[:, 0].abs() * 2.0 ** -7).sum()))
    return float(la) / 8, float(lt), ma, mt, ties


@pytest.mark.parametrize("capacity", [1, 3, 8])
def test_score_many_equals_each_utterance_alone(long_ctx, capacity):
    m, wd, cfg = long_ctx
    lengths = [150, 7, 40, 90, 3, 60, 128, 33, 200, 16, 1]
    items = _ragged_items(31, lengths)
    imp = InferenceImp(None, m, "teacher-force", 0.7, 25, 0.8, 30, "TTS")
    got = dict(imp.score_many(items, capacity=capacity))
    assert set(got) == {u for u, _, _ in items}
    for utt, seq, mask in items:
        r = got[utt]
        la, lt, ma, mt, ties = _alone(m, seq, mask)
        assert r["frames"] == seq.shape[1]
        for mine, ref in ((r["loss_audio"], la), (r["loss_text"], lt)):   # NaN (a group without any mask) on both sides
            assert (math.isnan(mine) and math.isnan(ref)) or abs(mine - ref) <= 1e-3 * abs(ref), (utt, mine, ref)
        na, nt = sum(row[1] for row in r["sums_audio"]), r["sums_text"][0][1]
        for key, ref, n, t in (("acc_all_audio", ma["acc_all"], na, ties[0]), ("acc_all_text", mt["acc_all"], nt, ties[1])):
            if n == 0:
                assert math.isnan(r[key]) and math.isnan(float(ref))
                continue
            assert abs(r[key] - float(ref)) * n <= t + 1e-3, (utt, key, r[key], float(ref), t)
    again = dict(imp.score_many(items, capacity=capacity))
    assert json.dumps(again, sort_keys=True) == json.dumps(got, sort_keys=True), "a repeated run gives identical results"
    # trailing frames whose mask is zero everywhere change nothing
    padded = [(u, torch.cat([s, torch.randint(0, 2048, (9, 5))], 1), torch.cat([k, torch.zeros(9, 5)], 1)) for u, s, k in items]
    assert json.dumps(dict(imp.score_many(padded, capacity=capacity)), sort_keys=True) == json.dumps(got, sort_keys=True)


def test_score_cli(tmp_path, gqa):
    from rstnet_b200 import offline
    m, wd, cfg = gqa
    c = _product_config(cfg)
    (tmp_path / "cfg.json").write_text(json.dumps(dataclasses.asdict(c)))
    torch.save({"model": {k: v.float().cpu() for k, v in m.state_dict().items()}}, tmp_path / "ck.pt")
    items = _ragged_items(7, [12, 5, 16])
    torch.save({u: {"seq": s, "mask": k} for u, s, k in items}, tmp_path / "corpus.pt")
    assert offline.main(["score", "--input", str(tmp_path / "corpus.pt"), "--config", str(tmp_path / "cfg.json"),
                         "--checkpoint", str(tmp_path / "ck.pt"), "--output-file", str(tmp_path / "o.json"),
                         "--capacity", "2"]) == 0
    out = json.loads((tmp_path / "o.json").read_text())
    assert set(out) == {"u0", "u1", "u2"} and all(math.isfinite(v["loss_audio"]) for v in out.values())
