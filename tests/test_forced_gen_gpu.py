"""Forced tokens during generation on the GPU (-m gpu): rstnet_lm_force_tokens against torch.where, forcing that agrees
with a run changing nothing (Moshi generate_many, GPT generate_many with fixed, windowed and best-of-N rows), greedy
LMGen.step(force=) against the oracle forced alike, rows without forcing untouched by forced rows next to them, and
`offline continue --force audio`."""
import dataclasses
import json

import numpy as np
import pytest
import torch

from oracle import lm_oracle as LO
from oracle import moshi_oracle as M
from rstnet_b200 import _lib, ops
from rstnet_b200.infer import InferenceImp
from rstnet_b200.lm import GPT, Config, _LMState
from rstnet_b200.moshi import LMGen, LMModel, generate_many, prompt_from_aligned

pytestmark = pytest.mark.gpu
DEV, BF = "cuda", torch.bfloat16
CFG = dataclasses.replace(M.SMALL, delays=(0, 0, 1, 2, 1, 0, 1, 2, 1, 0, 1, 2, 1, 0, 1, 2, 1))   # max_delay 2
K, DQ = CFG.n_q + 1, CFG.dep_q
N_USER = K - DQ - 1
MD = max(CFG.delays)
TEXT_EMPTY = 128002


# ------------------------------------------------------------------------------------------- 1. the kernel
@pytest.mark.parametrize("B", [1, 7, 64, 255, 256])
def test_force_tokens_equals_torch_where(B):
    L, st = _lib.lib(), ops._stream()
    g = torch.Generator().manual_seed(B)
    V, ts, fs = 300, DQ + 3, DQ + 2                      # row strides wider than the columns
    tokens0 = torch.randint(0, V, (B, ts), generator=g).to(DEV)
    force = torch.randint(-3, V, (B, fs), generator=g).to(torch.int32).to(DEV)
    _lib.lib().rstnet_device_error_flags(1)
    tokens = tokens0.clone()
    for col in range(DQ + 1):
        _lib.check(L.rstnet_lm_force_tokens(tokens.data_ptr(), ts, col, force.data_ptr(), fs, B, V, st))
    want = tokens0.clone()
    want[:, :DQ + 1] = torch.where(force[:, :DQ + 1] >= 0, force[:, :DQ + 1].long(), tokens0[:, :DQ + 1])
    assert torch.equal(tokens, want)
    assert _lib.lib().rstnet_device_error_flags(1) == 0
    # an id >= V: not written, error bit 1; the other rows of the launch still take theirs
    bad = force.clone()
    r = B // 2
    bad[r, 3] = V
    tokens = tokens0.clone()
    _lib.check(L.rstnet_lm_force_tokens(tokens.data_ptr(), ts, 3, bad.data_ptr(), fs, B, V, st))
    assert _lib.lib().rstnet_device_error_flags(1) & 1
    assert int(tokens[r, 3]) == int(tokens0[r, 3])
    ok = torch.arange(B, device=DEV) != r
    assert torch.equal(tokens[ok, 3], torch.where(bad[ok, 3] >= 0, bad[ok, 3].long(), tokens0[ok, 3]))


# ------------------------------------------------------------------------------------------- Moshi
@pytest.fixture(scope="module")
def moshi():
    w = M.synthetic_weights(CFG, seed=5)
    m = LMModel(**CFG.reference_kwargs())
    m.load_state_dict(w, strict=True)
    return m.to(DEV, BF).eval(), w


def _seq(L, seed):
    g = torch.Generator().manual_seed(seed)
    s = torch.randint(0, CFG.card, (K, L), generator=g)
    s[0] = torch.randint(0, CFG.text_card, (L,), generator=g)
    return s


def _corpus(n, seed, Pmax=20, Gmax=14):
    g = np.random.default_rng(seed)
    return [(f"u{i}", _seq(P + G, 1000 * seed + i), P)
            for i, (P, G) in enumerate((int(g.integers(0, Pmax)), int(g.integers(3, Gmax))) for _ in range(n))]


def _gen_all(m, items, capacity, **kw):
    gen = LMGen(m, use_sampling=True)
    return dict(generate_many(gen, items, capacity, seeds={u: 17 + int(u[1:]) for u, _, _ in items}, **kw))


def _observed(seq, P, out):
    """seq with Moshi's channels replaced by what the run output at every aligned frame it returned, and the mask of those
    frames -> (seq', observed bool [dep_q + 1, L])"""
    s, seen = seq.clone(), torch.zeros(DQ + 1, seq.shape[1], dtype=torch.bool)
    for j in range(out.shape[1]):
        f = P + j - MD
        if f >= 0:
            s[:DQ + 1, f] = out[:, j]
            seen[:, f] = True
    return s, seen


@pytest.mark.parametrize("paged", [False, True])
def test_moshi_forcing_that_agrees_changes_nothing(moshi, paged):
    """Every channel subset forced to what the unforced run produced: outputs bit-identical (each draw is keyed by the
    row's step, key and head, not by the other heads' tokens)."""
    m, _ = moshi
    items = _corpus(8, 3)
    kw = dict(kv_pages=40) if paged else {}
    base = _gen_all(m, items, 4, **kw)
    g = torch.Generator().manual_seed(1)
    items2, masks = [], {}
    for i, (u, seq, P) in enumerate(items):
        s, seen = _observed(seq, P, base[u])
        items2.append((u, s, P))
        pick = [seen & (torch.arange(DQ + 1)[:, None] == 0), seen & (torch.arange(DQ + 1)[:, None] > 0),
                seen & (torch.rand(seen.shape, generator=g) < 0.5), None][i % 4]
        if pick is not None:
            masks[u] = pick
    got = _gen_all(m, items2, 4, force=masks, **kw)
    assert set(got) == set(base)
    for u in base:
        assert torch.equal(got[u], base[u]), u


def test_moshi_unforced_rows_untouched(moshi):
    """Items forced to their recordings (which the model would not have drawn) next to items without forcing: the latter
    equal a run with no forcing at all, bit for bit, at the same capacity; every forced position holds the recording."""
    m, _ = moshi
    items = _corpus(7, 4)
    base = _gen_all(m, items, 3)
    masks = {u: torch.ones(DQ + 1, seq.shape[1], dtype=torch.bool) if i % 2 else
             (torch.arange(DQ + 1)[:, None] > 0).expand(DQ + 1, seq.shape[1]).clone()
             for i, (u, seq, _) in enumerate(items) if i % 3 != 2}
    got = _gen_all(m, items, 3, force=masks)
    seqs = {u: (s, P) for u, s, P in items}
    for u in base:
        if u not in masks:
            assert torch.equal(got[u], base[u]), u
            continue
        s, P = seqs[u]
        assert got[u].shape == base[u].shape
        for j in range(got[u].shape[1]):
            f = P + j - MD
            if f >= 0:
                k = masks[u][:, f]
                assert torch.equal(got[u][k, j], s[:DQ + 1, f][k]), (u, j)
    assert any(not torch.equal(got[u], base[u]) for u in masks)


def _margin(o, ours):
    _, _, text_logits, alog = o.last
    lt = text_logits.float()[:, 0, 0]
    return torch.cat([lt.max(-1).values - lt.gather(1, ours[:, :1])[:, 0],
                      (alog.float().max(-1).values - alog.float().gather(2, ours[:, 1:, None])[:, :, 0]).flatten()])


@pytest.mark.parametrize("paged", [False, True])
def test_forced_steps_vs_oracle(moshi, paged):
    """Greedy LMGen.step(force=) against LMGenOracle.step(force=): rows with the text forced, with the audio forced, a
    prompted row with its text forced, and a prompted row without forcing, admitted at different ticks.  Every forced
    token is the given id; every other decision is the oracle's argmax within the margin rule."""
    m, w = moshi
    B, T = 4, 14
    plan = {0: (0, 0, "text"), 1: (0, 0, "audio"), 2: (2, 7, "text"), 3: (1, 5, None)}   # row: (tick, P, forced)
    seqs = {r: _seq(P + T, 60 + r) for r, (_, P, _) in plan.items()}
    x = torch.randint(0, CFG.card, (T, B, N_USER, 1), generator=torch.Generator().manual_seed(9))
    g = torch.Generator().manual_seed(2)
    given = torch.randint(0, CFG.card, (T, B, DQ + 1), generator=g)
    given[:, :, 0] = torch.randint(0, CFG.text_card, (T, B), generator=g)
    gen = LMGen(m, use_sampling=False)
    wb = {k: v.to(BF) for k, v in w.items()}
    ora, stats = {}, {r: [0, 0, 0.0, 0] for r in plan}
    with gen.streaming(B, kv_pages=64 if paged else None), torch.no_grad():
        if paged:
            gen.reserve_kv(list(range(B)), 10 ** 6)
        for t in range(T):
            new = [r for r, (a, _, _) in plan.items() if a == t]
            if new:
                gen.reset_streaming(streams=new)
                prompts = {}
                for r in new:
                    P = plan[r][1]
                    prompts[r] = prompt_from_aligned(seqs[r], P, CFG.delays, DQ)
                    ora[r] = M.LMGenOracle(wb, CFG, 1)
                    for s in range(P):
                        ora[r].step(prompts[r][DQ + 1:, s].view(1, N_USER, 1), force=prompts[r][:DQ + 1, s].view(1, -1))
                gen.prefill_streams(prompts)
            force = torch.full((B, DQ + 1), -1, dtype=torch.int64)
            fmask = torch.zeros(B, DQ + 1, dtype=torch.bool)
            for r, (a, _, what) in plan.items():
                if a <= t and what is not None:
                    fmask[r] = torch.arange(DQ + 1) == 0 if what == "text" else torch.arange(DQ + 1) > 0
            force[fmask] = given[t][fmask]
            gen.step(x[t].to(DEV), force=force[:, :, None].to(DEV))
            tokens = gen._st.lm.tokens.cpu()
            assert torch.equal(tokens[fmask], force[fmask])
            for r, o in ora.items():
                ours = tokens[r:r + 1]
                o.step(x[t][r:r + 1], force=ours)
                d = _margin(o, ours)[~fmask[r]]
                stats[r][0] += int((d == 0).sum()); stats[r][1] += d.numel(); stats[r][2] = max(stats[r][2], float(d.max()))
                stats[r][3] += int(fmask[r].sum())
    assert _lib.lib().rstnet_device_error_flags(1) == 0
    for r, (exact, n, worst, nf) in stats.items():
        print(f"row {r} {plan[r]}: {exact}/{n} sampled decisions exact, worst deficit {worst:.3f}; {nf} forced")
        assert n > 0 and worst <= 0.1 and exact >= 0.8 * n
        assert (nf > 0) == (plan[r][2] is not None)


def test_offline_continue_force_audio(moshi, tmp_path):
    from rstnet_b200 import offline
    m, w = moshi
    cfg = tmp_path / "lm.json"
    cfg.write_text(json.dumps(CFG.reference_kwargs()))
    torch.save(w, tmp_path / "ckpt.pt")
    corpus = {f"d{i}": _seq(L, 300 + i) for i, L in enumerate([20, 30, 25])}
    torch.save(corpus, tmp_path / "corpus.pt")
    P = 8
    rc = offline.main(["continue", "--model", "moshi", "--config", str(cfg), "--checkpoint", str(tmp_path / "ckpt.pt"),
                       "--input", str(tmp_path / "corpus.pt"), "--prompt-frames", str(P), "--output-file",
                       str(tmp_path / "out.pt"), "--capacity", "2", "--seed", "3", "--force", "audio"])
    assert rc == 0
    out = torch.load(tmp_path / "out.pt")
    assert set(out) == set(corpus)
    for u, seq in corpus.items():
        o = out[u]
        assert o.shape == (DQ + 1, seq.shape[1] - P)
        for j in range(o.shape[1]):
            f = P + j - MD
            if f >= 0:
                assert torch.equal(o[1:, j], seq[1:DQ + 1, f]), (u, j)
    # the same as generate_many with the masks the CLI builds
    masks = {u: (torch.arange(DQ + 1)[:, None] > 0).expand(DQ + 1, s.shape[1]).clone() for u, s in corpus.items()}
    gen = LMGen(m, use_sampling=True, temp=0.8, temp_text=0.7, top_k=250, top_k_text=25)
    want = dict(generate_many(gen, [(u, s, P) for u, s in corpus.items()], 2, seeds={u: 3 for u in corpus}, force=masks))
    for u in want:
        assert torch.equal(out[u], want[u]), u


# ------------------------------------------------------------------------------------------- GPT batch TTS
@pytest.fixture(scope="module")
def lm():
    cfg = dataclasses.replace(LO.SMALL, context=128, block_size=512)
    w32 = LO.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05)
    m = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                   intermediate_size=cfg.intermediate_size, norm_eps=cfg.norm_eps, padded_vocab_size=cfg.padded_vocab_size,
                   audio_card=cfg.audio_card, n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim,
                   codecformer_heads=cfg.codecformer_heads, codecformer_layers=cfg.codecformer_layers,
                   codecformer_dim_feedforward=cfg.codecformer_dim_feedforward, context=cfg.context))
    m.load_state_dict(w32, strict=True)
    return m.to(DEV, BF).eval()


def _utt(P, G, seed):
    g = torch.Generator().manual_seed(seed)
    seq = torch.randint(0, 2048, (9, P + G), generator=g)
    seq[0, :P] = torch.randint(0, 1000, (P,), generator=g)
    seq[0, P:] = TEXT_EMPTY
    return seq


GCORPUS = [("a", _utt(20, 9, 1)), ("b", _utt(30, 16, 2)), ("c", _utt(12, 25, 3)), ("d", _utt(40, 6, 4)), ("e", _utt(9, 11, 5))]
GSEEDS = {"a": 3, "b": 11, "c": 5, "d": 0, "e": 8}
WINDOWS = {"b": (4, 20), "e": (-1, 15)}       # windowed rows: the stop rule applies from frame min + 1 on


def _imp(m):
    return InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")


def _frames_run(imp, **kw):
    return {u: (codes.cpu(), raw.cpu()) for u, codes, raw in
            imp.generate_many([(u, s.to(DEV)) for u, s in GCORPUS], 3, seeds=GSEEDS, lengths=WINDOWS, return_frames=True, **kw)}


def _G(u):
    """the frames item u may run: its window's max_frames, else its text-empty frames"""
    return WINDOWS[u][1] if u in WINDOWS else int((dict(GCORPUS)[u][0] == TEXT_EMPTY).sum())


def test_gpt_forcing_that_agrees_changes_nothing(lm):
    """Fixed and windowed rows: any subset of the generated frames' tokens forced to what the unforced run produced gives
    bit-identical frames and codes."""
    imp = _imp(lm)
    base = _frames_run(imp)
    g = torch.Generator().manual_seed(4)
    forced = {}
    for i, (u, _) in enumerate(GCORPUS):
        if i == 3:
            continue                                    # an item without forcing
        raw = base[u][1]                                # [G', 9]
        f = torch.full((9, _G(u)), -1, dtype=torch.int64)
        keep = torch.rand(raw.shape[1], raw.shape[0], generator=g) < (0.3, 1.0, 0.6, 0.6, 0.6)[i]
        f[:, :raw.shape[0]] = torch.where(keep, raw.t(), -1)
        forced[u] = f
    got = _frames_run(imp, forced=forced)
    assert set(got) == set(base)
    for u in base:
        assert torch.equal(got[u][0], base[u][0]) and torch.equal(got[u][1], base[u][1]), u


def test_gpt_best_of_n_forcing_that_agrees_changes_nothing(lm):
    """n_samples = 2: the candidates share the forced table, set where both candidates' codes agree; candidates, their
    codes, frame counts and log-probability sums are unchanged."""
    imp = _imp(lm)
    items = [(u, s.to(DEV)) for u, s in GCORPUS[:3]]
    run = lambda **kw: {u: c for u, c in imp.generate_many(items, 4, seeds=GSEEDS, lengths=WINDOWS, n_samples=2, **kw)}
    base = run()
    forced, n = {}, 0
    for u, cands in base.items():
        a, b = sorted(cands, key=lambda c: c.index)
        G = min(a.frames, b.frames)
        f = torch.full((9, _G(u)), -1, dtype=torch.int64)
        ca, cb = a.codes.cpu()[:, :G - 1], b.codes.cpu()[:, :G - 1]
        agree = ca == cb
        # codes[0, j] is audio codebook 0 of frame j, codes[l, j] codebook l of frame j + 1 (reverse_delay)
        f[1, :G - 1] = torch.where(agree[0], ca[0], -1)
        f[2:, 1:G] = torch.where(agree[1:], ca[1:], -1)
        forced[u] = f
        n += int((f >= 0).sum())
    assert n > 0
    got = run(forced=forced)
    for u in base:
        for x, y in zip(sorted(base[u], key=lambda c: c.index), sorted(got[u], key=lambda c: c.index)):
            assert torch.equal(x.codes.cpu(), y.codes.cpu()) and x.frames == y.frames, u
            assert x.logprob_audio == y.logprob_audio and x.logprob_text == y.logprob_text, u


def test_gpt_forced_rows_take_the_ids_and_others_are_untouched(lm, monkeypatch):
    """Utterances forced to ids the model would not draw (the semantic codebook fixed, ids inside the vocabulary but
    outside the candidate sets) take them; the unforced utterances of the batch equal a run without forcing, and only the
    forced frame graph is replayed."""
    imp = _imp(lm)
    base = _frames_run(imp)
    g = torch.Generator().manual_seed(6)
    forced = {}
    for u in ("a", "c"):
        f = torch.full((9, _G(u)), -1, dtype=torch.int64)
        f[1] = torch.randint(0, 2050, (_G(u),), generator=g)     # 2049 lies outside the 2048-id sets of later frames
        f[0, ::3] = torch.randint(0, 128004, (f[0, ::3].numel(),), generator=g)
        forced[u] = f
    keys = []
    orig = _LMState._replay
    monkeypatch.setattr(_LMState, "_replay", lambda self, key, fn: (keys.append(key), orig(self, key, fn))[1])
    got = _frames_run(imp, forced=forced)
    monkeypatch.setattr(_LMState, "_replay", orig)
    assert all("force" in k for k in keys if k[0] == "frame") and any(k[0] == "frame" for k in keys)
    for u in base:
        if u not in forced:
            assert torch.equal(got[u][1], base[u][1]), u
            continue
        raw = got[u][1]
        f = forced[u][:, :raw.shape[0]].t()
        assert torch.equal(raw[f >= 0], f[f >= 0]), u
    assert _lib.lib().rstnet_device_error_flags(1) == 0
