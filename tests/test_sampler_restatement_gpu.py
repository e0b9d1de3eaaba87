"""The LM sampler on the GPU (-m gpu) draw by draw against its host restatement (tests/sampler_restatement.py): every
token equals the restated draw or lies in its near-tie set, in every mode, at vocabulary sizes on both sides of the
candidate-list path, in the scalar and per-row table forms with the strides the LM uses, on crafted edge rows (ties at
the cuts, signed zeros, NaN, +-inf, subnormals, overflow), and in replays of the LM's own sampler calls."""
import dataclasses

import numpy as np
import pytest
import torch

import sampler_restatement as S
from oracle import sampling_oracle as O
from rstnet_b200 import _lib, ops
from rstnet_b200.lm import Sampling, _LMState

pytestmark = pytest.mark.gpu
DEV, BF = torch.device("cuda", 0), torch.bfloat16
CANARY = -7
NEAR_MAX = 0.02      # near-ties allowed per launch: a fraction of its rows (plus one)

TOP_K = [0, 1, 2, 63, 64, 65, 250, 1023, 1024, -1]
TEMP = [0.3, 0.7, 1.0, 1.5]
TOP_P = [0.0, 0.3, 0.9, 0.999999, 1.0]


def _i32(keys):
    k = [int(x) & 0xFFFFFFFF for x in keys]
    return torch.tensor([x - 2 ** 32 if x >= 2 ** 31 else x for x in k], dtype=torch.int32, device=DEV)


def launch(logits, top_k=0, temp=1.0, top_p=0.0, *, n_valid=0, nv_rows=None, tables=None, seed=1, step=None,
           step_rows=None, key_rows=None, tok_stride=9, nv_stride=2, prm_stride=2):
    """rstnet_lm_sample_params_bf16 with the LM's strides: tokens in column 0 of [R, tok_stride] (the other columns are
    canaries, checked untouched), per-row tables in column 0 of [R, stride]; -> int64 [R] on the host"""
    R, V = logits.shape
    tok = torch.full((R, tok_stride), CANARY, dtype=torch.int64, device=DEV)

    def table(vals, dtype, stride):
        t = torch.full((R, stride), -99, dtype=dtype)   # the other columns hold garbage the kernel must not read
        t[:, 0] = torch.as_tensor(np.asarray(vals), dtype=dtype)
        return t.to(DEV)
    tk = te = tp = None
    if tables is not None:
        tk, te, tp = (table(tables[0], torch.int32, prm_stride), table(tables[1], torch.float32, prm_stride),
                      table(tables[2], torch.float32, prm_stride))
    nv = None if nv_rows is None else table(nv_rows, torch.int32, nv_stride)
    sc = None if step is None else torch.tensor([step], dtype=torch.int64, device=DEV)
    sr = None if step_rows is None else torch.as_tensor(step_rows, dtype=torch.int64).to(DEV)
    kr = None if key_rows is None else _i32(key_rows)
    p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    _lib.check(_lib.lib().rstnet_lm_sample_params_bf16(
        logits.data_ptr(), R, V, n_valid, p(nv), nv_stride, top_k, float(temp), float(top_p), p(tk), p(te), p(tp), prm_stride,
        seed, p(sc), p(sr), p(kr), tok.data_ptr(), tok_stride, ops._stream()), "sample_params")
    tok = tok.cpu()
    assert bool((tok[:, 1:] == CANARY).all()), "the sampler wrote outside its token column"
    return tok[:, 0]


def check(tok, draws, what, near_max=NEAR_MAX):
    """every token in [0, n_valid) and in its restated set; -> the number of near-ties (printed, and bounded)"""
    near = 0
    for r, (t, d) in enumerate(zip(tok.tolist(), draws)):
        assert t in d.ok, (what, r, d.mode, t, sorted(d.ok)[:8])
        near += not d.exact
    assert near <= near_max * len(draws) + 1, (what, near, len(draws))
    print(f"{what}: {len(draws)} rows, {near} near-ties")
    return near


def both(logits, top_k=0, temp=1.0, top_p=0.0, **kw):
    """launch and restate the same arguments; -> (tokens, restated draws); every token in [0, n_valid)"""
    tok = launch(logits, top_k, temp, top_p, **kw)
    kw = {k: v for k, v in kw.items() if k not in ("tok_stride", "nv_stride", "prm_stride")}
    draws = S.draw_launch(logits.cpu(), top_k=top_k, temp=temp, top_p=top_p, **kw)
    nv = [S.resolve(logits.shape[1], kw.get("n_valid", 0), 0, 1.0, 0.0,
                    None if kw.get("nv_rows") is None else kw["nv_rows"][r]).n_valid for r in range(len(tok))]
    assert all(0 <= t < n for t, n in zip(tok.tolist(), nv)), "a token outside [0, n_valid)"
    return tok, draws


KINDS = ["gumbel", "coarse", "tail", "planted"]


def rows_of_kinds(R, V, seed=0):
    """R bf16 logit rows [R, V] on the device: the sampling oracle's kinds in turn, at scales 0.5 .. 2"""
    return torch.stack([O.logit_row(seed + r, V, KINDS[r % 4], (0.5, 1.0, 2.0)[r % 3], temp=0.7, p=0.9)
                        for r in range(R)]).to(DEV)


def _tables(R, salt):
    """every (top_k, temp, top_p) combination in turn (200), started at a salt"""
    combos = [(k, t, p) for p in TOP_P for t in TEMP for k in TOP_K]
    sel = [combos[(salt + 7 * r) % len(combos)] for r in range(R)]
    return tuple(list(c) for c in zip(*sel))


# ------------------------------------------------------------------------------------------------ 1. shapes x settings
SHAPES = [(8, 300), (2050, 300), (4096, 256), (4097, 256), (32000, 37), (152064, 37)]


@pytest.mark.parametrize("V,R", SHAPES)
def test_per_row_tables_every_setting(V, R):
    """Mixed modes per row from the settings tables, per-row candidate counts on both sides of V (and 4096 / 4097 for
    the list path), and the per-row RNG with steps past 2^32 and keys past 2^31."""
    lg = rows_of_kinds(R, V, seed=V)
    nv = [(V, V - 1, max(V // 2 + 1, 1), 0, V + 5, 4096, 4097)[r % 7] for r in range(R)]
    total = 0
    for salt, seed in ((0, 0), (3, 2 ** 32 - 1)):
        sr = [2 ** 32 + 3 * r + salt if r % 2 else r for r in range(R)]
        kr = [2 ** 31 + 5 * r if r % 3 == 0 else 11 * r + 1 for r in range(R)]
        tok, draws = both(lg, nv_rows=nv, tables=_tables(R, salt), seed=seed, step_rows=sr, key_rows=kr)
        total += check(tok, draws, f"tables V={V} seed={seed}")
    assert total <= NEAR_MAX * 2 * R + 1


@pytest.mark.parametrize("V,R", [(8, 37), (4097, 37), (152064, 4)])
@pytest.mark.parametrize("top_k", TOP_K)
def test_scalar_form_every_top_k(V, R, top_k):
    """the scalar form with the scope counter (a step past 2^32 truncates to its low 32 bits) at each top_k, with a
    temperature and nucleus setting by turns"""
    lg = rows_of_kinds(R, V, seed=3 * V + top_k)
    temp, top_p = TEMP[top_k % 4], TOP_P[(top_k + 7) % 5]
    tok, draws = both(lg, top_k, temp, top_p, n_valid=V - 1 if V > 8 else 0, seed=2 ** 32 - 1, step=2 ** 32 + 9)
    check(tok, draws, f"scalar V={V} top_k={top_k}")
    # the counter's low 32 bits key the noise: a step of 9 draws the same tokens
    assert torch.equal(launch(lg, top_k, temp, top_p, n_valid=V - 1 if V > 8 else 0, seed=2 ** 32 - 1, step=9), tok)


# ------------------------------------------------------------------------------------------------ 2. crafted rows
def _row(V, fill=-1e4):
    return torch.full((V,), fill, dtype=torch.float32)


def signed_zero_row(V):
    """+0 at id 0, -0 at ids 1..3, 64 tiny positive logits further on, the rest far below"""
    r = _row(V, -30.0)
    r[0] = 0.0
    r[1:4] = -0.0
    r[100:164] = 1e-30 * torch.arange(1, 65)
    return r


def zero_ties_row(V):
    """+0 and -0 interleaved at random ids: the threshold order must not put every +0 before a lower -0"""
    r = torch.randn(V, generator=torch.Generator().manual_seed(V)) - 6.0
    ids = torch.randperm(V, generator=torch.Generator().manual_seed(1))[:600]
    r[ids] = torch.where(torch.arange(600) % 2 == 0, torch.tensor(0.0), torch.tensor(-0.0))
    r[ids[:20]] = 1.0
    return r


def tie_row(V, n_ties, lead=5.0):
    """a few leading logits, then n_ties equal ones at spread-out ids (the top-k and nucleus cuts fall among them)"""
    r = _row(V)
    r[:3] = torch.tensor([lead, lead - 0.5, lead - 1.0])
    ids = torch.linspace(3, V - 1, n_ties).long()
    r[ids] = 1.0
    return r


def three_ties_row(V):
    """three equal logits and nothing else: nucleus p = 0.5 keeps exactly the first two (mass before 0, 1/3 <= 1/2)"""
    r = _row(V, float("-inf"))
    r[[V // 5, V // 2, V - 2]] = 0.25
    return r


def nan_row(V):
    r = torch.randn(V, generator=torch.Generator().manual_seed(V + 1))
    r[torch.arange(0, V, 7)] = float("nan")
    r[1] = 9.0          # a NaN (id 0) and the largest finite logit side by side
    r[0] = float("nan")
    return r


def nan_ties_row(V):
    """NaN at ids 0..9 (positive and negative: 0x7FC0, 0xFFC1) and 70 equal logits at ids 10..79: top_k = 64 or 66
    keeps the first 64 or 66 of the ties; a NaN that took a top-k slot would drop the last ones (bf16 [V])"""
    r = _row(V)
    r[10:80] = 1.0
    r = r.to(BF)
    bits = r.view(torch.int16)
    bits[:5] = 0x7FC0
    bits[5:10] = 0xFFC1 - 0x10000
    return r


def crafted(V):
    """name -> bf16 row [V] (V > 164)"""
    out = {
        "signed_zeros": signed_zero_row(V), "zero_ties": zero_ties_row(V), "ties_few": tie_row(V, min(300, V - 3)),
        "three_ties": three_ties_row(V), "nan": nan_row(V), "nan_ties": nan_ties_row(V),
        "one_pos_inf": torch.where(torch.arange(V) == V // 3, torch.tensor(float("inf")), torch.randn(V)),
        "all_neg_inf": _row(V, float("-inf")), "all_nan": _row(V, float("nan")),
        "nan_and_neg_inf": torch.where(torch.arange(V) % 2 == 0, torch.tensor(float("nan")), torch.tensor(float("-inf"))),
        "subnormal": torch.randn(V, generator=torch.Generator().manual_seed(5)) * 2.0 ** -130,
        "huge": torch.where(torch.arange(V) % 3 == 0, torch.tensor(3e38), torch.tensor(-3e38)) * torch.where(
            torch.arange(V) % 5 == 0, -1.0, 1.0),
    }
    if V > 2100:
        out["ties_many"] = tie_row(V, 2000)
    return {k: v.to(BF) for k, v in out.items()}


@pytest.mark.parametrize("V", [2050, 4097, 152064])
def test_crafted_rows_every_mode(V):
    """Each crafted row over 64 noise keys in each mode.  Ties at the top-k cut (fewer and more than SAMPLE_CAND of
    them) and at the nucleus cut are taken lowest index first; -0 ties +0; NaN is never drawn nor takes a top-k slot;
    a row with no id above -inf draws 0."""
    R = 64
    rows = crafted(V)
    modes = [(0, 1.0, 0.0), (1, 0.7, 0.0), (2, 1.0, 0.0), (64, 1.0, 0.0), (66, 1.0, 0.0), (250, 0.7, 0.0), (1024, 1.0, 0.0),
             (-1, 0.3, 0.0), (-1, 1.0, 0.5), (5, 0.7, 0.3), (-1, 1.5, 0.999999)]
    for name, row in rows.items():
        lg = row.to(DEV).expand(R, -1).contiguous()
        tab = tuple(list(c) for c in zip(*[modes[r % len(modes)] for r in range(R)]))
        for seed in (0, 2 ** 32 - 1):
            kw = dict(tables=tab, seed=seed, step_rows=[r // len(modes) for r in range(R)], key_rows=list(range(R)))
            tok, draws = both(lg, **kw)
            check(tok, draws, f"{name} V={V} seed={seed}", near_max=0.1)


@pytest.mark.parametrize("V", [2050, 4097, 152064])
def test_signed_zeros_at_the_top_k_cut(V):
    """+0 at id 0, -0 at ids 1..3 and 64 tiny positive logits (all of about equal weight): top_k = 66 keeps the 64, the
    +0 and the -0 at id 1, top_k = 65 no -0.  The threshold select must rank -0 and +0 as one value: ordering -0 below
    +0 counted the +0 twice and kept 65 ids.  On 1024 noise keys id 1 is drawn with top_k >= 66, id 2 with 67."""
    R = 1024
    lg = signed_zero_row(V).to(BF).to(DEV).expand(R, -1).contiguous()
    x = S._values(lg[0].cpu(), V)
    assert set(S.topk_set(x, 66).tolist()) == set(range(100, 164)) | {0, 1}
    kw = dict(step_rows=[0] * R, key_rows=list(range(R)), seed=7)
    for k in (65, 66, 67):
        tok, draws = both(lg, k, 1.0, 0.0, **kw)
        check(tok, draws, f"signed zeros top_k={k}")
        assert (1 in tok.tolist()) == (k >= 66), k
        assert (2 in tok.tolist()) == (k >= 67), k


def test_ties_at_the_nucleus_cut():
    """three equal logits at p = 0.5: the first two ids are kept and drawn about evenly, the third never"""
    for V in (2050, 152064):
        R = 256
        lg = three_ties_row(V).to(BF).to(DEV).expand(R, -1).contiguous()
        tok, draws = both(lg, -1, 1.0, 0.5, step_rows=[3] * R, key_rows=list(range(R)), seed=9)
        check(tok, draws, f"three ties V={V}", near_max=0.0)
        c = np.bincount(tok.numpy(), minlength=V)
        assert c[V // 5] > 64 and c[V // 2] > 64 and c[V - 2] == 0, (c[V // 5], c[V // 2], c[V - 2])


def test_rows_without_a_candidate_draw_zero():
    """every mode on all -inf, all NaN and NaN/-inf rows, also past n_valid: id 0, never the 0x7fffffff sentinel"""
    for V in (8, 4097, 152064):
        rows = {"all_neg_inf": _row(V, float("-inf")), "all_nan": _row(V, float("nan")),
                "nan_and_neg_inf": torch.where(torch.arange(V) % 2 == 0, torch.tensor(float("nan")), torch.tensor(float("-inf")))}
        for name, row in rows.items():
            lg = row.to(BF).to(DEV).expand(len(TOP_K) * 2, -1).contiguous()
            tab = ([k for k in TOP_K for _ in range(2)], [0.7] * 20, [0.0, 0.9] * 10)
            tok = launch(lg, tables=tab, step_rows=[1] * 20, key_rows=list(range(20)))
            assert tok.tolist() == [0] * 20, (V, name, tok.tolist())
            for tk in TOP_K:
                assert launch(lg[:2], tk, 0.7, 0.0, step=2).tolist() == [0, 0], (V, name, tk)
                assert launch(lg[:2], tk, 0.7, 0.9, step=2).tolist() == [0, 0], (V, name, tk)


# ------------------------------------------------------------------------------------------------ 3. the LM's own draws
def _spy(monkeypatch, rec):
    """record each _LMState._sample call: its logits, parameters, RNG key and the column it drew"""
    orig = _LMState._sample

    def spy(self, col, mode, n_valid, per_row_rng):
        torch.cuda.synchronize()
        c = self.c
        V = c.padded_vocab_size if col == 0 else c.audio_card
        logits = (self.logits if col == 0 else self.dlogits).reshape(-1, V)[:self.M].cpu()
        r = dict(col=col, logits=logits, seed=self.seed + col, mode=mode, n_valid=n_valid)
        if mode is None:
            h = min(col, 1)
            r["tables"] = (self.row_topk[:self.M, h].tolist(), self.row_temp[:self.M, h].tolist(),
                           self.row_topp[:self.M, h].tolist())
        if n_valid is None:
            r["nv_rows"] = self.row_valid[:self.M, col - 1].tolist()
        if per_row_rng:
            r["step_rows"] = self.row_step[:self.M].tolist()
            r["key_rows"] = [k & 0xFFFFFFFF for k in self.row_key[:self.M].tolist()]
        else:
            r["step"] = int(self.frame_counter.item())
        orig(self, col, mode, n_valid, per_row_rng)
        torch.cuda.synchronize()
        r["tok"] = self.tokens[:self.M, col].cpu()
        rec.append(r)

    monkeypatch.setattr(_LMState, "_sample", spy)


def replay(rec, what):
    """each recorded call under the restatement"""
    assert rec
    n = near = 0
    for r in rec:
        tk, temp, tp = r["mode"] if r["mode"] is not None else (0, 1.0, 0.0)
        draws = S.draw_launch(r["logits"], n_valid=r["n_valid"] or 0, top_k=tk, temp=temp, top_p=tp,
                              nv_rows=r.get("nv_rows"), tables=r.get("tables"), seed=r["seed"], step=r.get("step"),
                              step_rows=r.get("step_rows"), key_rows=r.get("key_rows"))
        for row, (t, d) in enumerate(zip(r["tok"].tolist(), draws)):
            assert t in d.ok, (what, r["col"], row, t, sorted(d.ok)[:8], d.mode)
            near += not d.exact
        n += len(draws)
    print(f"{what}: {len(rec)} sampler calls, {n} rows, {near} near-ties")
    assert near <= NEAR_MAX * n + 1
    return rec


@pytest.fixture(scope="module")
def small_lm():
    """L.SMALL with context 128, as test_tts_best_of_gpu.py"""
    from oracle import lm_oracle as L
    from rstnet_b200.lm import GPT, Config
    cfg = dataclasses.replace(L.SMALL, context=128, block_size=512)
    w32 = L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05)
    m = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                   intermediate_size=cfg.intermediate_size, norm_eps=cfg.norm_eps, padded_vocab_size=cfg.padded_vocab_size,
                   audio_card=cfg.audio_card, n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim,
                   codecformer_heads=cfg.codecformer_heads, codecformer_layers=cfg.codecformer_layers,
                   codecformer_dim_feedforward=cfg.codecformer_dim_feedforward, context=cfg.context))
    m.load_state_dict(w32, strict=True)
    return m.to(DEV, BF).eval()


def test_generate_many_draws_replayed(small_lm, monkeypatch):
    """generate_many with per-row settings (argmax, top-k, nucleus, multinomial), rows admitted at different frames
    (capacity 3 for 7 utterances of different lengths) and a best-of-3 request: every draw of every head"""
    from test_tts_batch_gpu import _corpus
    from rstnet_b200.infer import InferenceImp
    m = small_lm
    corpus = _corpus(7, 21, pmax=12, gmax=6)
    kinds = [Sampling(use_sampling=False), Sampling(top_k_text=25, top_k=30, temp=1.3), Sampling(top_p_text=0.9, top_p=0.8),
             Sampling(top_k_text=0, top_k=0, temp_text=0.5), Sampling(top_k_text=300, top_k=100, temp=0.6)]
    sampling = {u: kinds[i % len(kinds)] for i, (u, _) in enumerate(corpus)}
    seeds = {u: (2 ** 32 - 3 + 5 * i) & 0xFFFFFFFF for i, (u, _) in enumerate(corpus)}
    imp = InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")
    rec = []
    _spy(monkeypatch, rec)
    m.use_cuda_graphs = False
    try:
        got = dict(imp.generate_many(((u, s.to(DEV)) for u, s in corpus), 3, seeds=seeds, sampling=sampling))
        assert len(got) == len(corpus)
        n_plain = len(rec)
        best = list(imp.generate_many([corpus[1]], 3, seeds=seeds, sampling=sampling, n_samples=3))
        assert len(best) == 1 and len(rec) > n_plain
    finally:
        m.use_cuda_graphs = True
    assert any(r.get("tables") for r in rec) and any(r.get("step_rows") for r in rec)
    replay(rec, "generate_many")


def test_lmgen_draws_replayed(monkeypatch):
    """LMGen steps of the Moshi model with per-session settings and seeds, a session restarted mid-run"""
    from oracle import moshi_oracle as M
    from rstnet_b200.moshi import LMGen, LMModel
    w = M.synthetic_weights(M.SMALL, seed=5)
    lm = LMModel(**M.SMALL.reference_kwargs())
    lm.load_state_dict(w, strict=True)
    lm = lm.to(DEV, BF).eval()
    lm.use_cuda_graphs = False
    n_user = M.SMALL.n_q - M.SMALL.dep_q
    sess = [Sampling(top_p=0.85, top_p_text=0.9, temp=1.0), Sampling(use_sampling=False), Sampling(top_k=5, temp=1.4),
            Sampling(top_k=0, top_k_text=0), Sampling(top_k=100, top_k_text=70, temp=0.5)]
    rec = []
    _spy(monkeypatch, rec)
    B = len(sess)
    for per_row in (True, False):
        gen = LMGen(lm, use_sampling=True, temp=0.8, top_k=250)
        with gen.streaming(B):
            if per_row:
                for r in range(B):
                    gen.set_stream_sampling([r], sess[r], seed=(2 ** 31 + 977 * r) if r % 2 else r)
            for t in range(8):
                if per_row and t == 4:
                    gen.reset_streaming(streams=[2])
                    gen.set_stream_sampling([2], sess[0], seed=2 ** 32 - 1)
                x = torch.randint(0, M.SMALL.card, (B, n_user, 1), generator=torch.Generator().manual_seed(t)).to(DEV)
                gen.step(x)
    assert any(r.get("step_rows") for r in rec) and any(r.get("step") is not None for r in rec)
    replay(rec, "LMGen")
