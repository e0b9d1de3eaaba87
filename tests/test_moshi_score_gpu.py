"""GPU tests (-m gpu) of Moshi scoring: the pair-RoPE append's row-map entry point against uniform launches, the
non-streaming forward_text / forward against the reference's outputs (tests/golden/moshi_score.npz), moshi.score_many
against scoring each utterance alone, and forward inside an LMGen scope."""
import json
import math
import os

import numpy as np
import pytest
import torch

import moshi_score_oracle as O
from oracle import moshi_oracle as M
from rstnet_b200 import _lib
from rstnet_b200.lm import MAX_ROWS, CrossEntropyAndAccuracy
from rstnet_b200.moshi import LMGen, LMModel, score_many

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16


def _cos(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float(torch.dot(a, b) / (a.norm() * b.norm()).clamp(min=1e-12))


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-6))


# ------------------------------------------------------------------------------------------------ the kernel
@pytest.mark.parametrize("hd", [64, 128])
def test_rows_entry_point_equals_uniform_launches(hd):
    """A shuffled row map with padding rows writes the q_out rows and ring bytes of a uniform launch of the same (stream,
    position) pairs, bit for bit, with positions past 2^24; padding rows and pairs left out touch nothing."""
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    B, H, T, cap = 3, 4, 7, 11
    g = torch.Generator().manual_seed(hd)
    off = torch.tensor([0, (1 << 24) + 5, 3 * (1 << 24) + 17], dtype=torch.int64, device=DEV)
    freqs = torch.exp(torch.arange(hd // 2, dtype=torch.float32) * (-math.log(10000.0) * 2 / hd)).to(DEV)
    qkv_u = (torch.randn(T * B, 3, H, hd, generator=g) * 2).to(BF).to(DEV)
    canary = (torch.randn(2, B, H, cap, hd, generator=g) * 7).to(BF).to(DEV)
    q_u = torch.full((T * B, H * hd), 3.5, dtype=BF, device=DEV)
    kv_u = canary.clone()
    _lib.check(lib.rstnet_lm_rope_pair_kv_append_bf16(qkv_u.data_ptr(), off.data_ptr(), 1, q_u.data_ptr(), kv_u.data_ptr(), T * B, B,
                                                      H, hd, cap, freqs.data_ptr(), st))
    # the mapped launch: every pair of streams 0 and 2, stream 1's first 4 positions (the ring has room for all of them),
    # shuffled, with padding rows between
    pairs = [(b, t) for t in range(T) for b in (0, 2)] + [(1, t) for t in range(4)]
    perm = torch.randperm(len(pairs), generator=g).tolist()
    rows = []
    for i, p in enumerate(perm):
        rows.append(pairs[p])
        if i % 5 == 2:
            rows.append((-1, 0))
    rows.append((-1, 3))
    R = len(rows)
    rs = torch.tensor([b for b, _ in rows], dtype=torch.int32, device=DEV)
    rt = torch.tensor([t for _, t in rows], dtype=torch.int32, device=DEV)
    qkv_m = (torch.randn(R, 3, H, hd, generator=g) * 2).to(BF).to(DEV)   # padding rows keep their noise
    for r, (b, t) in enumerate(rows):
        if b >= 0:
            qkv_m[r] = qkv_u[t * B + b]
    q_m = torch.full((R, H * hd), 3.5, dtype=BF, device=DEV)
    kv_m = canary.clone()
    _lib.check(lib.rstnet_lm_rope_pair_kv_append_rows_bf16(qkv_m.data_ptr(), off.data_ptr(), rs.data_ptr(), rt.data_ptr(),
                                                           q_m.data_ptr(), kv_m.data_ptr(), R, B, H, hd, cap, freqs.data_ptr(), st))
    torch.cuda.synchronize()
    for r, (b, t) in enumerate(rows):
        if b < 0:
            assert bool((q_m[r] == 3.5).all()), "a padding row writes no q_out"
        else:
            assert torch.equal(q_m[r], q_u[t * B + b]), (r, b, t)
    want = canary.clone()
    for b, t in pairs:
        slot = (int(off[b]) + t) % cap
        want[:, b, :, slot] = kv_u[:, b, :, slot]
    assert torch.equal(kv_m.view(torch.int16), want.view(torch.int16)), "ring bytes: written pairs as uniform, the rest untouched"


# ------------------------------------------------------------------------------------------------ the model
@pytest.fixture(scope="module")
def moshi(golden_dir):
    from oracle.gen_golden import weights_digest
    cfg = M.SMALL
    w = M.synthetic_weights(cfg, seed=5)
    gold = np.load(os.path.join(golden_dir, "moshi_score.npz"))
    assert weights_digest(w) == str(gold["weights_sha256"])
    m = LMModel(**cfg.reference_kwargs())
    m.load_state_dict(w, strict=True)
    return m.to(DEV, BF).eval(), {k: v.to(BF) for k, v in w.items()}, cfg, gold


def test_forward_text_and_forward_vs_reference_golden(moshi):
    """S = 40 > context = 16: our bf16 deviation from an fp32 evaluation of the same bf16 weights <= 2x the reference's."""
    m, wd, cfg, gold = moshi
    seqs, masks = torch.from_numpy(gold["seqs"]), torch.from_numpy(gold["masks"])
    B, K, S = seqs.shape
    assert S > cfg.context
    w32 = {k: v.float() for k, v in wd.items()}
    with torch.no_grad():
        t_audio, t_text = O.forward(w32, cfg, seqs)
    tc, ac = torch.from_numpy(gold["text_cols"]), torch.from_numpy(gold["audio_cols"])
    # forward_text outside a scope, on the forward's own input sequence
    start = torch.full((B, K, 1), cfg.card, dtype=torch.long)
    start[:, 0] = cfg.text_card
    inputs = torch.cat([start, seqs[:, :, :-1]], 2)
    out, tl = m.forward_text(inputs.to(DEV))
    assert out.shape == (B, S, cfg.dim) and tl.shape == (B, 1, S, cfg.text_card) and out.dtype == tl.dtype == BF
    ref_text = torch.from_numpy(gold["bf16_text_logits"])
    truth_text = t_text.float()[..., tc]
    mine = tl[:, 0].float().cpu()[..., tc]
    assert _cos(mine, ref_text) >= 0.999
    assert _rel(mine, truth_text) <= 2.0 * _rel(ref_text, truth_text) + 1e-2, (_rel(mine, truth_text), _rel(ref_text, truth_text))
    audio, text = m(seqs.to(DEV), masks.to(DEV))
    assert audio.shape == (B, S, cfg.dep_q, cfg.card) and text.shape == (B, S, cfg.text_card)
    assert torch.equal(text, tl[:, 0]), "forward's text logits are forward_text's"
    ref_audio = torch.from_numpy(gold["bf16_audio_logits"])
    truth_audio = t_audio.float()[..., ac]
    mine = audio.float().cpu()[..., ac]
    assert _cos(mine, ref_audio) >= 0.999
    assert _rel(mine, truth_audio) <= 2.0 * _rel(ref_audio, truth_audio) + 1e-2, (_rel(mine, truth_audio), _rel(ref_audio, truth_audio))
    # the metrics of validate_model on our logits: within the reference's own bf16 distance of the fp32 truth (x2)
    met = CrossEntropyAndAccuracy(audio, seqs[:, 1:9].to(DEV), masks[:, 1:9].to(DEV), O.AUDIO_WEIGHTS, [O.IGNORE_AUDIO] * 8)[1]
    t_met = O.validate(t_audio, t_text, seqs, masks)
    ref = float(gold["bf16_loss_audio"])
    assert abs(float(met["loss"]) - float(t_met["loss_audio"])) <= 2.0 * abs(ref - float(t_met["loss_audio"])) + 1e-3 * abs(ref)


def _items(cfg, seed, lengths):
    g = torch.Generator().manual_seed(seed)
    K = cfg.n_q + 1
    items = []
    for j, Lj in enumerate(lengths):
        seq = torch.randint(0, cfg.card, (K, Lj), generator=g)
        seq[0] = torch.randint(0, cfg.text_card, (Lj,), generator=g)
        pick = torch.rand(K, Lj, generator=g)
        seq[1:][pick[1:] < 0.05] = O.IGNORE_AUDIO
        seq[0][pick[0] < 0.05] = O.IGNORE_TEXT
        mask = torch.tensor([0.0, 0.5, 1.0, 1.0, 1.0])[torch.randint(0, 5, (K, Lj), generator=g)]
        if j == 2:
            mask[1 + 5] = 0.0                                    # an audio codebook masked out throughout: NaN loss
        items.append((f"u{j}", seq, mask))
    return items


def _alone(m, seq, mask):
    """validate_model's metrics of LMModel.forward on one utterance, and the rows whose bf16 top-2 margin is within one
    bf16 step of the maximum (rounding may flip their argmax)."""
    audio, text = m(seq[None].to(DEV))
    s, mk = seq[None].to(DEV), mask[None].to(DEV)
    la, ma = CrossEntropyAndAccuracy(audio, s[:, 1:9], mk[:, 1:9], O.AUDIO_WEIGHTS, [O.IGNORE_AUDIO] * 8)
    lt, mt = CrossEntropyAndAccuracy(text.unsqueeze(2), s[:, 0].unsqueeze(1), mk[:, 0:1], [1], [O.IGNORE_TEXT])
    ties = []
    for lg in (audio.float().reshape(-1, audio.shape[-1]), text.float().reshape(-1, text.shape[-1])):
        t2 = lg.topk(2, dim=-1).values
        ties.append(int(((t2[:, 0] - t2[:, 1]) <= t2[:, 0].abs() * 2.0 ** -7).sum()))
    return float(la), float(lt), ma, mt, ties


@pytest.mark.parametrize("capacity", [1, 3, 8])
def test_score_many_equals_each_utterance_alone(moshi, capacity):
    m, wd, cfg, gold = moshi
    lengths = [1, 300, 40, MAX_ROWS + 9, 7, 3 * cfg.context, 90, 2, 200, 16, 17]   # 1 frame, > MAX_ROWS, > context
    items = _items(cfg, 31, lengths)
    got = dict(score_many(m, items, capacity=capacity))
    assert set(got) == {u for u, _, _ in items}
    for utt, seq, mask in items:
        r = got[utt]
        la, lt, ma, mt, ties = _alone(m, seq, mask)
        assert r["frames"] == seq.shape[1]
        for mine, ref in ((r["loss_audio"], la), (r["loss_text"], lt)):
            assert (math.isnan(mine) and math.isnan(ref)) or abs(mine - ref) <= 1e-3 * abs(ref), (utt, mine, ref)
        na, nt = sum(row[1] for row in r["sums_audio"]), r["sums_text"][0][1]
        for key, ref, n, t in (("acc_audio", ma["acc_all"], na, ties[0]), ("acc_text", mt["acc_all"], nt, ties[1])):
            if n == 0:
                assert math.isnan(r[key]) and math.isnan(float(ref))
                continue
            assert abs(r[key] - float(ref)) * n <= t + 1e-3, (utt, key, r[key], float(ref), t)
    assert math.isnan(got["u2"]["loss_audio"]) and math.isfinite(got["u1"]["loss_audio"])
    again = dict(score_many(m, items, capacity=capacity))
    assert json.dumps(again, sort_keys=True) == json.dumps(got, sort_keys=True), "a repeated run gives identical results"
    padded = [(u, torch.cat([s, torch.randint(0, cfg.card, (s.shape[0], 5))], 1), torch.cat([k, torch.zeros(k.shape[0], 5)], 1))
              for u, s, k in items]
    assert json.dumps(dict(score_many(m, padded, capacity=capacity)), sort_keys=True) == json.dumps(got, sort_keys=True)


def test_forward_inside_lmgen_scope_raises_and_changes_nothing(moshi):
    m, wd, cfg, gold = moshi
    B = 2
    g = torch.Generator().manual_seed(3)
    inputs = [torch.randint(0, cfg.card, (B, cfg.n_q - cfg.dep_q, 1), generator=g).to(DEV) for _ in range(6)]
    seq = torch.from_numpy(gold["seqs"]).to(DEV)
    gen = LMGen(m, use_sampling=False)

    def run(interrupt):
        outs = []
        with gen.streaming(B):
            for t, inp in enumerate(inputs):
                if interrupt and t == 3:
                    with pytest.raises(_lib.RstnetError):
                        m(seq)
                r = gen.step(inp)
                outs.append(None if r is None else r.cpu())
        return outs
    plain, interrupted = run(False), run(True)
    assert all((a is None and b is None) or torch.equal(a, b) for a, b in zip(plain, interrupted))


def test_score_cli_moshi(tmp_path, moshi):
    from rstnet_b200 import offline
    m, wd, cfg, gold = moshi
    (tmp_path / "lm.json").write_text(json.dumps(cfg.reference_kwargs()))
    torch.save({k: v.float().cpu() for k, v in m.state_dict().items()}, tmp_path / "ck.pt")
    items = _items(cfg, 7, [12, 5, 30])
    torch.save({u: {"seq": s, "mask": k} for u, s, k in items}, tmp_path / "corpus.pt")
    assert offline.main(["score", "--model", "moshi", "--input", str(tmp_path / "corpus.pt"), "--config", str(tmp_path / "lm.json"),
                         "--checkpoint", str(tmp_path / "ck.pt"), "--output-file", str(tmp_path / "o.json"),
                         "--capacity", "2"]) == 0
    out = json.loads((tmp_path / "o.json").read_text())
    direct = dict(score_many(m, items, capacity=2))
    assert json.dumps(out, sort_keys=True) == json.dumps(direct, sort_keys=True)
