"""Nucleus (top-p) sampling and per-row sampling settings on the GPU (-m gpu): rstnet_lm_sample_params_bf16 against the
reference's kept sets (tests/golden/sampling_top_p.npz) and the float64 restatement (oracle/sampling_oracle.py), its exact
relations to the multinomial and between its per-row and scalar forms, and the per-row settings through GPT.forward_step,
InferenceImp.generate_many and LMGen."""
import os

import numpy as np
import pytest
import torch

from oracle import sampling_oracle as O
from oracle.gen_golden_sampling import row_logits
from rstnet_b200 import _lib, ops
from rstnet_b200.lm import Sampling

pytestmark = pytest.mark.gpu
DEV, BF = torch.device("cuda", 0), torch.bfloat16
MARGIN = 3e-5   # as tests/test_sampling_params_cpu.py: the reference's fp32 cumsum against float64


def _i32(keys):
    """uint32 keys as their int32 bits on the device"""
    k = [int(x) & 0xFFFFFFFF for x in keys]
    return torch.tensor([x - 2 ** 32 if x >= 2 ** 31 else x for x in k], dtype=torch.int32, device=DEV)


def params(logits, top_k=0, temp=1.0, top_p=0.0, *, n_valid=0, nv_rows=None, tables=None, seed=1, step=None, step_rows=None,
           key_rows=None):
    """rstnet_lm_sample_params_bf16 on logits [R, V]; tables = (top_k [R], temp [R], top_p [R]); -> int64 [R] on the host"""
    R, V = logits.shape
    out = torch.zeros(R, dtype=torch.int64, device=DEV)
    tk = te = tp = None
    if tables is not None:
        tk = torch.as_tensor(tables[0], dtype=torch.int32).to(DEV)
        te = torch.as_tensor(tables[1], dtype=torch.float32).to(DEV)
        tp = torch.as_tensor(tables[2], dtype=torch.float32).to(DEV)
    nv = None if nv_rows is None else torch.as_tensor(nv_rows, dtype=torch.int32).to(DEV)
    sc = None if step is None else torch.tensor([step], dtype=torch.int64, device=DEV)
    sr = None if step_rows is None else torch.as_tensor(step_rows, dtype=torch.int64).to(DEV)
    kr = None if key_rows is None else _i32(key_rows)
    p = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    _lib.check(_lib.lib().rstnet_lm_sample_params_bf16(logits.data_ptr(), R, V, n_valid, p(nv), 1, top_k, float(temp), float(top_p),
                                                       p(tk), p(te), p(tp), 1, seed, p(sc), p(sr), p(kr), out.data_ptr(), 1,
                                                       ops._stream()), "sample_params")
    return out.cpu()


def fixture():
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sampling_top_p.npz"))
    for j in range(len(g["seed"])):
        r = (int(g["seed"][j]), int(g["V"][j]), int(g["n_valid"][j]), str(g["kind"][j]), float(g["scale"][j]),
             float(g["temp"][j]), float(g["p"][j]))
        yield r, np.unpackbits(g["kept_bits"][j])[:r[2]].astype(bool), row_logits(*r)


# ------------------------------------------------------------------------------------------------ 1. kept sets
def test_draws_lie_in_the_reference_kept_set():
    """Every fixture row, 64 rows of draws (per-row keys) x 4 steps: each draw is in the float64 kept set widened by the
    margin, and its logit is at least the smallest logit the reference kept."""
    for (seed, V, n_valid, kind, scale, temp, p), ref_keep, lg in fixture():
        R = 64
        rows = lg.to(DEV).expand(R, -1).contiguous()
        wide = O.kept_set(lg, n_valid, temp, p, MARGIN)
        lo = float(lg[:n_valid].float()[torch.from_numpy(ref_keep)].min())
        for step in range(4):
            tok = params(rows, -1, temp, p, n_valid=n_valid, step_rows=[step] * R, key_rows=list(range(R)), seed=seed)
            assert bool((tok >= 0).all() and (tok < n_valid).all()), (seed, kind)
            assert wide[tok.numpy()].all(), (seed, V, kind, p)
            assert float(lg.float()[tok].min()) >= lo, (seed, V, kind, p)


def test_crafted_row_ratio():
    """probabilities 0.40 / 0.35 / 0.25 at p = 0.5: the first two in a 40:35 ratio, the third never"""
    V = 3
    lg = torch.tensor([np.log(0.40), np.log(0.35), np.log(0.25)], dtype=torch.float32)
    rows = lg.to(BF).to(DEV).expand(4096, -1).contiguous()
    w = torch.softmax(lg.to(BF).double(), 0)[:2]
    counts = np.zeros(V)
    for step in range(4):
        tok = params(rows, -1, 1.0, 0.5, step_rows=[step] * 4096, key_rows=list(range(4096)), seed=3)
        counts += np.bincount(tok.numpy(), minlength=V)
    assert counts[2] == 0
    assert abs(counts[0] / counts.sum() - float(w[0] / w.sum())) < 1.5e-2


# ------------------------------------------------------------------------------------------------ 2. exact relations
@pytest.mark.parametrize("V", [2050, 152064])
def test_nucleus_relations_to_multinomial(V):
    """(a) p >= the whole mass (0.999999 on a flat row, where every id is kept): the multinomial draw bit for bit;
    (b) at any p, whenever the multinomial draw is in the nucleus, the nucleus draw equals it."""
    R = 128
    lg = O.logit_row(9, V, "gumbel", 0.6).to(DEV).expand(R, -1).contiguous()
    flat = torch.zeros(R, V, dtype=BF, device=DEV)
    kw = dict(step_rows=list(range(R)), key_rows=[7 * r for r in range(R)], seed=11)
    assert torch.equal(params(flat, -1, 1.0, 0.999999, **kw), params(flat, -1, 1.0, 0.0, **kw))
    assert torch.equal(params(lg, -1, 0.9, 1.0, **kw), params(lg, -1, 0.9, 0.0, **kw))
    row = lg[0].cpu()
    for p in (0.3, 0.8, 0.95):
        keep = O.kept_set(row, V, 0.9, p, -MARGIN)
        multi = params(lg, -1, 0.9, 0.0, **kw)
        nuc = params(lg, -1, 0.9, p, **kw)
        inside = torch.from_numpy(keep[multi.numpy()])
        assert bool(inside.any())
        assert torch.equal(nuc[inside], multi[inside]), p


def test_empirical_distribution_matches_nucleus():
    """the reference's self-test criterion (utils/sampling.py:157-175): |empirical - renormalised nucleus| < 1.5e-2"""
    V, temp, p = 64, 1.0, 0.8
    lg = O.logit_row(4, V, "gumbel", 1.0)
    rows = lg.to(DEV).expand(1024, -1).contiguous()
    counts = np.zeros(V)
    for step in range(4):
        counts += np.bincount(params(rows, -1, temp, p, step_rows=[step] * 1024, key_rows=list(range(1024)), seed=5).numpy(),
                              minlength=V)
    assert np.abs(counts / counts.sum() - O.kept_probs(lg, V, temp, p)).max() < 1.5e-2


# ------------------------------------------------------------------------------------------------ 4./5. per-row tables
@pytest.mark.parametrize("top_k,temp", [(0, 1.0), (1, 0.8), (25, 0.7), (64, 1.1), (65, 0.8), (250, 0.8), (1024, 1.0), (-1, 0.8)])
def test_uniform_table_equals_scalar_form(top_k, temp):
    """a settings table holding one setting draws what the scalar settings draw, with per-row candidate counts and RNG;
    and the per-row RNG keyed (step s, row r) and the one-setting table draw what the scope counter at s draws"""
    R, V = 12, 2050
    g = torch.Generator().manual_seed(top_k + 2)
    lg = torch.randn(R, V, generator=g).mul(2).to(BF).to(DEV)
    nv = [2048, 2049, 2050, 2048] * 3
    kr, sr = [3 * r + 1 for r in range(R)], [r % 5 for r in range(R)]
    table = lambda n: ([top_k] * n, [temp] * n, [0.0] * n)   # noqa: E731
    want = params(lg, top_k, temp, 0.0, nv_rows=nv, step_rows=sr, key_rows=kr)
    got = params(lg, 0, 1.0, 0.0, nv_rows=nv, tables=table(R), step_rows=sr, key_rows=kr)
    assert torch.equal(got, want)
    # the scalar form with the scope counter
    want = params(lg, top_k, temp, 0.0, n_valid=2049, step=6)
    assert torch.equal(params(lg, top_k, temp, 0.0, n_valid=2049, step_rows=[6] * R, key_rows=list(range(R))), want)
    assert torch.equal(params(lg, n_valid=2049, tables=table(R), step=6), want)
    text = torch.randn(4, 152064, generator=g).to(BF).to(DEV)
    want = params(text, top_k, temp, 0.0, step=2)
    assert torch.equal(params(text, top_k, temp, 0.0, step_rows=[2] * 4, key_rows=list(range(4))), want)
    assert torch.equal(params(text, tables=table(4), step=2), want)


def test_mixed_modes_per_row():
    modes = [(0, 1.0, 0.0), (25, 0.7, 0.0), (250, 0.9, 0.0), (-1, 0.8, 0.0), (-1, 0.8, 0.9), (30, 1.2, 0.5), (-1, 1.0, 1.0),
             (64, 0.6, 0.0)]
    R = len(modes) * 3
    g = torch.Generator().manual_seed(8)
    lg = torch.randn(R, 32000, generator=g).mul(1.5).to(BF).to(DEV)
    sr, kr = [r * 2 for r in range(R)], [100 + r for r in range(R)]
    tab = [modes[r % len(modes)] for r in range(R)]
    got = params(lg, tables=tuple(zip(*tab)), step_rows=sr, key_rows=kr)
    for r in range(R):
        tk, te, tp = tab[r]
        alone = params(lg[r:r + 1].contiguous(), tk, te, tp, step_rows=sr[r:r + 1], key_rows=kr[r:r + 1])
        assert int(got[r]) == int(alone[0]), (r, tab[r])


# ------------------------------------------------------------------------------------------------ 6./7. determinism, edges
def test_identical_calls_and_graph_replays_give_identical_bytes():
    R, V = 32, 152064
    lg = O.logit_row(21, V, "coarse", 1.0).to(DEV).expand(R, -1).contiguous()
    kw = dict(step_rows=[0] * R, key_rows=list(range(R)), seed=2)
    first = params(lg, -1, 0.8, 0.9, **kw)
    for _ in range(3):
        assert torch.equal(params(lg, -1, 0.8, 0.9, **kw), first)
    out = torch.zeros(R, dtype=torch.int64, device=DEV)
    sr = torch.zeros(R, dtype=torch.int64, device=DEV)
    kr = _i32(list(range(R)))
    L = _lib.lib()

    def launch():
        _lib.check(L.rstnet_lm_sample_params_bf16(lg.data_ptr(), R, V, 0, None, 1, -1, 0.8, 0.9, None, None, None, 1, 2, None,
                                                  sr.data_ptr(), kr.data_ptr(), out.data_ptr(), 1, ops._stream()))
    launch()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        launch()
    for _ in range(3):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.cpu(), first)


def test_inf_tails_and_massive_ties_at_the_cut():
    V = 152064
    # -inf tail: nothing past the finite ids is drawn
    tail = O.logit_row(31, V, "tail", 1.0)
    R = 64
    tok = params(tail.to(DEV).expand(R, -1).contiguous(), -1, 1.0, 0.99, step_rows=[1] * R, key_rows=list(range(R)))
    assert bool((tok < V // 2).all())
    # 3 000 equal logits under one top id holding 10% of the mass at temp 1: p = 0.5 keeps the top id and the first
    # ties by index up to mass 0.5 (walk of more than 1 024 ties); only ids from that prefix are drawn
    row = torch.full((V,), -1e4, dtype=torch.float32)
    ties = torch.arange(1000, 1000 + 3 * 3000, 3)
    row[ties] = 0.0
    row[5] = float(np.log(0.1 / 0.9 * 3000))
    rows = row.to(BF).to(DEV).expand(R, -1).contiguous()
    keep = O.kept_set(row.to(BF), V, 1.0, 0.5)
    for step in range(3):
        tok = params(rows, -1, 1.0, 0.5, step_rows=[step] * R, key_rows=list(range(R)))
        assert keep[tok.numpy()].all()
    n_ties_kept = int(keep[ties.numpy()].sum())
    assert 1024 < n_ties_kept < 3000
    assert keep[ties[:n_ties_kept].numpy()].all() and not keep[ties[n_ties_kept:].numpy()].any()
    # all candidates -inf but one; a single candidate
    one = torch.full((2, 2050), float("-inf"), dtype=BF, device=DEV)
    one[:, 17] = 0.0
    assert params(one, -1, 0.7, 0.5, step=0).tolist() == [17, 17]
    assert params(torch.randn(3, 2050, dtype=BF, device=DEV), -1, 0.7, 0.5, n_valid=1, step=0).tolist() == [0, 0, 0]


def test_host_validation():
    lg = torch.zeros(1, 16, dtype=BF, device=DEV)
    for bad in (dict(top_k=2000), dict(top_k=5, temp=0.0), dict(top_p=-0.1), dict(top_p=float("nan")), dict(top_p=float("inf"))):
        with pytest.raises(_lib.RstnetError):
            params(lg, **{"temp": 1.0, **bad})
    out = torch.zeros(1, dtype=torch.int64, device=DEV)
    t = torch.zeros(1, dtype=torch.int32, device=DEV)
    with pytest.raises(_lib.RstnetError):      # tables go together
        _lib.check(_lib.lib().rstnet_lm_sample_params_bf16(lg.data_ptr(), 1, 16, 0, None, 1, 0, 1.0, 0.0, t.data_ptr(), None, None, 1,
                                                           1, None, None, None, out.data_ptr(), 1, ops._stream()))


# ------------------------------------------------------------------------------------------------ layers
@pytest.fixture(scope="module")
def small_lm():
    """L.SMALL as in test_tts_batch_gpu.py"""
    from oracle import lm_oracle as L
    from rstnet_b200.lm import GPT, Config
    cfg = L.SMALL
    w32 = L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05)
    m = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                   intermediate_size=cfg.intermediate_size, norm_eps=cfg.norm_eps, padded_vocab_size=cfg.padded_vocab_size,
                   audio_card=cfg.audio_card, n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim,
                   codecformer_heads=cfg.codecformer_heads, codecformer_layers=cfg.codecformer_layers,
                   codecformer_dim_feedforward=cfg.codecformer_dim_feedforward, context=cfg.context))
    m.load_state_dict(w32, strict=True)
    m.use_cuda_graphs = True
    return m.to(DEV, BF).eval()


SETTINGS = {
    "argmax": Sampling(use_sampling=False),
    "topk": Sampling(top_k_text=25, top_k=30),
    "topp": Sampling(top_p_text=0.9, top_p=0.8, temp=1.0),
    "multi": Sampling(top_k_text=0, top_k=0, temp_text=1.0),
}


def test_generate_many_mixed_settings_equal_each_utterance_alone(small_lm):
    from test_tts_batch_gpu import _corpus
    from rstnet_b200.infer import InferenceImp
    m = small_lm
    corpus = _corpus(10, 9)
    names = list(SETTINGS)
    chosen = {u: SETTINGS[names[i % len(names)]] for i, (u, _) in enumerate(corpus)}
    seeds = {u: 1000 + i for i, (u, _) in enumerate(corpus)}
    alone = {}
    for utt, seq in corpus:
        imp = InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")
        s = chosen[utt]
        imp.use_sampling, imp.temp_text, imp.top_k_text, imp.top_p_text = s.use_sampling, s.temp_text, s.top_k_text, s.top_p_text
        imp.temp, imp.top_k, imp.top_p = s.temp, s.top_k, s.top_p
        got = dict(imp.generate_many([(utt, seq.to(DEV))], 1, seeds=seeds))
        alone[utt] = got[utt].cpu()
    imp = InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")
    for cap in (1, 4, 7):
        got = dict(imp.generate_many(((u, s.to(DEV)) for u, s in corpus), cap, seeds=seeds, sampling=chosen))
        for utt, codes in got.items():
            assert torch.equal(codes.cpu(), alone[utt]), (cap, utt)


def test_generate_with_top_p_equals_generate_many_alone(small_lm):
    """generate() (scalar settings, scope counter) and generate_many (per-row tables, key 0) draw the same codes"""
    from test_tts_batch_gpu import _corpus
    from rstnet_b200.infer import InferenceImp
    m = small_lm
    imp = InferenceImp(None, m, "sampling", 0.7, 25, 1.0, 30, "TTS")
    imp.top_p, imp.top_p_text = 0.8, 0.9
    for utt, seq in _corpus(3, 4):
        a = imp.generate(seq.unsqueeze(0).to(DEV))[0].cpu()
        b = dict(imp.generate_many([(utt, seq.to(DEV))], 3, sampling={utt: imp.sampling()}))[utt].cpu()
        c = dict(imp.generate_many([(utt, seq.to(DEV))], 2))[utt].cpu()
        assert torch.equal(a, b) and torch.equal(a, c), utt


def test_forward_step_per_row_equals_scalar_and_captures_no_new_graph(small_lm):
    m = small_lm
    B, dq = 4, m.config.dep_q
    g = torch.Generator().manual_seed(3)
    frames = [torch.randint(0, 2048, (B, 9, 1), generator=g).to(DEV) for _ in range(6)]
    valid = torch.full((B, dq), 2049, dtype=torch.int32)
    keys = [5, 6, 7, 8]
    for s in SETTINGS.values():
        runs = []
        for per_row in (False, True):
            with m.streaming(B):
                out = []
                for t, f in enumerate(frames):
                    kw = dict(sampling=[s] * B) if per_row else dict(
                        use_sampling=s.use_sampling, temp_text=s.temp_text, top_k_text=s.top_k_text, top_p_text=s.top_p_text,
                        temp=s.temp, top_k=s.top_k, top_p=s.top_p)
                    out.append(m.forward_step(f, audio_valid=valid, sample_key=keys if t == 0 else None, depth_ring_quirk=False, **kw))
                runs.append(torch.stack(out).cpu())
        assert torch.equal(runs[0], runs[1])
    with m.streaming(B):
        names = list(SETTINGS)
        for t, f in enumerate(frames * 2):
            m.forward_step(f, audio_valid=valid, sampling=[SETTINGS[names[(t + r) % 4]] for r in range(B)], depth_ring_quirk=False)
            if t == 3:
                n_graphs = len(m._state.graphs)
        assert len(m._state.graphs) == n_graphs


def test_lmgen_session_independent_of_row_and_tick():
    """A row given its own settings and seed draws the same tokens whichever row it runs in and whenever it starts, next
    to rows with other settings."""
    from oracle import moshi_oracle as M
    from rstnet_b200.moshi import LMGen, LMModel
    w = M.synthetic_weights(M.SMALL, seed=5)
    lm = LMModel(**M.SMALL.reference_kwargs())
    lm.load_state_dict(w, strict=True)
    lm = lm.to(DEV, BF).eval()
    n_user = M.SMALL.n_q - M.SMALL.dep_q
    inp = torch.randint(0, M.SMALL.card, (12, n_user), generator=torch.Generator().manual_seed(1))
    mine = Sampling(top_p=0.85, top_p_text=0.9, temp=1.0)
    others = [Sampling(use_sampling=False), Sampling(top_k=5), Sampling(top_k=0, top_k_text=0)]

    def run(B, row, start):
        gen = LMGen(lm, use_sampling=True, temp=0.8, top_k=250)
        outs = []
        with gen.streaming(B):
            for r in range(B):
                gen.set_stream_sampling([r], others[r % 3], seed=50 + r)
            mask = np.ones(B, dtype=np.int64)
            mask[row] = 0
            for t in range(start + 10):
                if t == start:
                    gen.reset_streaming(streams=[row])
                    gen.set_stream_sampling([row], mine, seed=1234)
                    mask[row] = 1
                gen.set_active_streams(mask)
                x = torch.randint(0, M.SMALL.card, (B, n_user, 1), generator=torch.Generator().manual_seed(t)).to(DEV)
                if t >= start:
                    x[row, :, 0] = inp[t - start].to(DEV)
                o = gen.step(x)
                if t >= start and gen.valid_rows()[row]:
                    outs.append(o[row, :, 0].cpu())
        return torch.stack(outs)

    a = run(3, 0, 0)
    assert torch.equal(a, run(3, 2, 3))
    assert torch.equal(a, run(3, 1, 5))
