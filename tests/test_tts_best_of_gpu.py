"""Best-of-N TTS on the GPU (-m gpu): rstnet_kv_pages_copy against torch indexing, generate_many(n_samples=N) candidates
against each candidate's seed run alone (with copy-on-write at a ring wrap and with admissions that wait for pages), the
in-frame log-probabilities against a float64 log_softmax of the frame's own logits and against a teacher-forced
GPT.forward, the plain frame graph left as it is, and suspend / resume of a forked row."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from oracle import lm_oracle as L
from rstnet_b200 import _lib, ops, row_state
from rstnet_b200.infer import InferenceImp, sample_seed
from rstnet_b200.lm import GPT, Config, Sampling, _LMState

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
BF = torch.bfloat16
TEXT_EMPTY = 128002


# ------------------------------------------------------------------------------------------------ 1. the page copy
def _copy(pools, pairs, page_bytes, ctas=8):
    ptrs = (C.c_void_p * len(pools))(*[p.data_ptr() for p in pools])
    return _lib.lib().rstnet_kv_pages_copy(ptrs, len(pools), pairs.data_ptr(), pairs.shape[0], page_bytes, ctas, ops._stream())


def _expect(pools, pairs):
    out = [p.clone() for p in pools]
    if len(pairs):
        pr = pairs.cpu().long()
        for o in out:
            o[pr[:, 1]] = o[pr[:, 0]]
    return out


@pytest.mark.parametrize("page_bytes", [4096, 2 * 64 * 128 * 2, 4099, 1030, 12])
@pytest.mark.parametrize("n_pairs", [1, 7])
@pytest.mark.parametrize("where", ["device", "pinned"])
def test_kv_pages_copy_byte_exact(page_bytes, n_pairs, where):
    g = torch.Generator().manual_seed(page_bytes + n_pairs)
    n_pages, n_pools = 20, 3
    pools = [torch.randint(0, 256, (n_pages, page_bytes), generator=g, dtype=torch.uint8).to(DEV) for _ in range(n_pools)]
    perm = torch.randperm(n_pages, generator=g)
    src, dst = perm[:n_pairs], perm[n_pairs:2 * n_pairs]
    if n_pairs > 1:
        src[1] = src[0]                    # one page copied to two places
    pairs = torch.stack([src, dst], 1).to(torch.int32).contiguous()
    pairs = pairs.to(DEV) if where == "device" else pairs.pin_memory()
    want = _expect(pools, pairs)
    n0 = _lib.launch_count()
    _lib.check(_copy(pools, pairs, page_bytes), "kv_pages_copy")
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0 + 1
    for a, b in zip(pools, want):
        assert torch.equal(a, b)


def test_kv_pages_copy_misaligned_pool_base_and_graph_capture():
    page_bytes = 256
    base = torch.randint(0, 256, (3, 10 * page_bytes + 1), dtype=torch.uint8).to(DEV)
    pools = [base[i, 1:].view(10, page_bytes) for i in range(3)]      # base address odd: byte accesses
    pairs = torch.tensor([[0, 5], [2, 7]], dtype=torch.int32).pin_memory()
    want = _expect(pools, pairs)
    _lib.check(_copy(pools, pairs, page_bytes), "kv_pages_copy")
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(pools, want))
    # captured with a pinned host table: every replay reads the table's entries as they are then
    aligned = [torch.randint(0, 256, (12, 1024), dtype=torch.uint8).to(DEV) for _ in range(2)]
    tab = torch.tensor([[1, 3], [4, 9]], dtype=torch.int32).pin_memory()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        graph = ops.capture(lambda: _lib.check(_copy(aligned, tab, 1024), "kv_pages_copy"))
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    want = _expect(aligned, tab)
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(aligned, want))
    tab[0, 0], tab[0, 1] = 10, 11
    want = _expect(aligned, tab)
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(aligned, want))


@pytest.mark.parametrize("where", ["device", "pinned"])
def test_kv_pages_copy_errors_launch_nothing(where):
    pools = [torch.randint(0, 256, (8, 64), dtype=torch.uint8).to(DEV) for _ in range(2)]
    snap = [p.clone() for p in pools]
    lib = _lib.lib()
    n0 = _lib.launch_count()
    bad = {"negative page": [[0, 1], [-1, 2]], "onto itself": [[3, 3]], "the dst of two pairs": [[0, 4], [1, 4]],
           "both a src and a dst": [[0, 1], [1, 2]]}
    for msg, pr in bad.items():
        t = torch.tensor(pr, dtype=torch.int32)
        t = t.to(DEV) if where == "device" else t.pin_memory()
        assert _copy(pools, t, 64) != 0, msg
        assert msg in lib.rstnet_last_error().decode(), (msg, lib.rstnet_last_error())
    unpinned = torch.tensor([[0, 1]], dtype=torch.int32)
    assert _copy(pools, unpinned, 64) != 0 and "neither device memory nor pinned" in lib.rstnet_last_error().decode()
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert all(torch.equal(a, b) for a, b in zip(pools, snap))


# ------------------------------------------------------------------------------------------------ 2. best-of-N TTS
@pytest.fixture(scope="module")
def lm():
    """L.SMALL with context 128 (two KV pages of 64 positions per ring) and block_size 512: a prompt of more than one page
    shares a full page, and P + G > 128 reaches it again at the ring wrap."""
    cfg = dataclasses.replace(L.SMALL, context=128, block_size=512)
    w32 = L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05)
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


# (P, G): inside one page, across pages with a shared full page, and past the ring (copy-on-write of page 0)
CORPUS = [("a", _utt(20, 9, 1)), ("b", _utt(70, 12, 2)), ("c", _utt(100, 40, 3)), ("d", _utt(64, 70, 4))]
SEEDS = {"a": 3, "b": 11, "c": 2 ** 32 - 5, "d": 0}
PROMPT = {"a": 20, "b": 70, "c": 100, "d": 64}


def _imp(m):
    return InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")


def _alone(imp, utt, seq, seed, cap, kv_pages, sampling):
    got = list(imp.generate_many([(utt, seq.to(DEV))], cap, seeds={utt: seed}, kv_pages=kv_pages,
                                 sampling=None if sampling is None else {utt: sampling}))
    assert len(got) == 1
    return got[0][1].cpu()


@pytest.mark.parametrize("n", [1, 2, 4])
@pytest.mark.parametrize("kv_pages", [None, 10])
def test_candidates_equal_their_seed_run_alone(lm, n, kv_pages, monkeypatch):
    imp = _imp(lm)
    sampling = {"b": Sampling(temp=1.1, top_k=0, top_p=0.9), "d": Sampling(use_sampling=False)}
    cap = 8
    cows = []
    orig = _LMState.copy_pages
    monkeypatch.setattr(_LMState, "copy_pages", lambda self, pairs: (pairs and cows.append(len(pairs)), orig(self, pairs))[1])
    stats = {}
    got = list(imp.generate_many(((u, s.to(DEV)) for u, s in CORPUS), cap, seeds=SEEDS, kv_pages=kv_pages, sampling=sampling,
                                 stats=stats, n_samples=n))
    monkeypatch.setattr(_LMState, "copy_pages", orig)
    assert sorted(u for u, _ in got) == sorted(u for u, _ in CORPUS)
    if kv_pages is not None and n == 4:
        assert stats["wait_frames"] > 0            # "c" and "d" need 8 of the 10 pages each: admissions wait
    seqs = dict(CORPUS)
    for utt, res in got:
        if n == 1:
            assert torch.equal(res.cpu(), _alone(imp, utt, seqs[utt], SEEDS[utt], cap, kv_pages, sampling.get(utt)))
            continue
        assert sorted(c.index for c in res) == list(range(n))
        key = [(-c.logprob_audio / c.frames, c.index) for c in res]
        assert key == sorted(key)                  # ranked by mean audio log-probability per frame, ties by index
        for c in res:
            assert c.frames == seqs[utt].shape[1] - PROMPT[utt]
            want = _alone(imp, utt, seqs[utt], sample_seed(SEEDS[utt], c.index), cap, kv_pages, sampling.get(utt))
            assert torch.equal(c.codes.cpu(), want), (utt, c.index)
            assert np.isfinite(c.logprob_audio) and c.logprob_audio < 0 and np.isfinite(c.logprob_text)
    if n > 1:
        # the forks' partial-page copies and, for "c" and "d" (P + G > 128), the copies of page 0 at the wrap
        assert len(cows) > len(CORPUS)


def test_plain_graph_untouched(lm, monkeypatch):
    """generate_many without n_samples and with n_samples=1: the same codes, stats and graph keys, none with logprob"""
    imp = _imp(lm)
    runs = []
    for kw in ({}, {"n_samples": 1}):
        keys = []
        orig = _LMState._replay
        monkeypatch.setattr(_LMState, "_replay", lambda self, key, fn: (keys.append(key), orig(self, key, fn))[1])
        stats = {}
        codes = {u: c.cpu() for u, c in imp.generate_many(((u, s.to(DEV)) for u, s in CORPUS), 3, seeds=SEEDS, stats=stats, **kw)}
        monkeypatch.setattr(_LMState, "_replay", orig)
        runs.append((codes, stats, keys))
    (c0, s0, k0), (c1, s1, k1) = runs
    assert s0 == s1 and k0 == k1 and c0.keys() == c1.keys()
    assert all(torch.equal(c0[u], c1[u]) for u in c0)
    frame_keys = {k for k in k0 if k[0] == "frame"}
    assert frame_keys == {("frame", ((25, 0.7, 0.0), (30, 0.8, 0.0)), "rows", True, False)}, frame_keys


@pytest.mark.parametrize("top_k,top_p", [(0, 0.0), (-1, 0.0), (5, 0.0), (-1, 0.9)])
def test_sampler_draws_only_ids_the_logits_cover(top_k, top_p):
    """The in-frame log-probability takes each sampled id as a label of its head's logits: the sampler clamps a candidate
    count above V (a scalar or a per-row table) to V, so no id >= V is ever drawn, even where the largest logits lie at
    the end of the row."""
    rows, V = 64, 40
    logits = torch.linspace(-2.0, 6.0, V).repeat(rows, 1).to(DEV, BF).contiguous()
    nv = torch.full((rows,), 2049, dtype=torch.int32, device=DEV)
    for n_valid, table in ((V + 9, None), (V, nv)):
        tok = torch.full((rows, 2), -7, dtype=torch.int64, device=DEV)
        _lib.check(_lib.lib().rstnet_lm_sample_params_bf16(
            logits.data_ptr(), rows, V, n_valid, None if table is None else table.data_ptr(), 1, top_k, 1.5, top_p, None, None,
            None, 2, 99, None, None, None, tok.data_ptr(), 2, ops._stream()), "sample")
        torch.cuda.synchronize()
        assert bool(((tok[:, 0] >= 0) & (tok[:, 0] < V)).all()), tok[:, 0]


def test_logprob_equals_float64_log_softmax_of_the_frame_logits(lm, monkeypatch):
    """Each candidate's sums against a float64 log_softmax of the logits the frame sampled from (recorded eagerly, without
    graphs), at the ids it sampled: only the fp32 per-row terms and fp64 sums differ."""
    imp = _imp(lm)
    N = 4
    rec = []
    orig = _LMState._logprob

    def spy(self, col):
        logits = self.logits if col == 0 else self.dlogits
        rec.append((col, logits.double().clone(), self.tokens[:, col].clone(), self.lp_slot.clone()))
        orig(self, col)

    monkeypatch.setattr(_LMState, "_logprob", spy)
    lm.use_cuda_graphs = False
    try:
        utt, cands = next(imp.generate_many([("b", CORPUS[1][1].to(DEV))], N, seeds=SEEDS, n_samples=N))
    finally:
        lm.use_cuda_graphs = True
    want = torch.zeros(N, 9, dtype=torch.float64)
    for col, logits, tok, slot in rec:
        assert bool(((tok >= 0) & (tok < logits.shape[1])).all())   # every sampled id is covered by its head
        lp = torch.log_softmax(logits, -1).gather(1, tok[:, None])[:, 0].cpu()
        act = slot.cpu() >= 0
        want[act, col] += lp[act]
    assert len(rec) == 9 * CORPUS[1][1].shape[1] - 9 * 70
    for c in cands:
        a, t = want[c.index, 1:].sum().item(), want[c.index, 0].item()
        assert abs(c.logprob_audio - a) <= 1e-6 * abs(a) + 1e-4, (c.index, c.logprob_audio, a)
        assert abs(c.logprob_text - t) <= 1e-6 * abs(t) + 1e-4, (c.index, c.logprob_text, t)


def test_logprob_agrees_with_teacher_forced_forward(lm, monkeypatch):
    """Against GPT.forward over [prompt, generated frames]: the same model, but the temporal transformer runs as one
    non-streaming pass instead of one step per frame, so the bf16 logits differ by rounding.  The bound on the mean
    difference per sampled token was measured on the H100 (see TF_TOL)."""
    imp = _imp(lm)
    N, P = 2, 70
    seq = CORPUS[1][1]
    utt, cands = next(imp.generate_many([("b", seq.to(DEV))], N, seeds=SEEDS, n_samples=N))
    diffs = []
    for c in cands:   # each candidate's frames: its seed run alone (equal codes: test_candidates_equal_their_seed_run_alone)
        _, raw = next((u, r) for u, _, r in imp.generate_many([("b", seq.to(DEV))], N, seeds={"b": sample_seed(SEEDS["b"], c.index)},
                                                              return_frames=True))
        full = torch.cat([seq[:, :P], raw.cpu().t()], 1)[None]       # [1, 9, P + G]
        audio_logits, text_logits = lm(full.to(DEV))
        g = torch.arange(P, P + c.frames)
        lt = torch.log_softmax(text_logits[0, g].double(), -1).gather(1, full[0, 0, g].to(DEV)[:, None]).sum().item()
        la = torch.log_softmax(audio_logits[0, g].double(), -1).gather(2, full[0, 1:, g].t().to(DEV)[:, :, None]).sum().item()
        n_tok = c.frames * 8
        diffs.append((abs(c.logprob_audio - la) / n_tok, abs(c.logprob_text - lt) / c.frames))
    for da, dt in diffs:
        assert da <= TF_TOL and dt <= TF_TOL, diffs


# mean |difference| per sampled token between the in-frame sums and the teacher-forced recomputation.  The two paths run
# the same bf16 model but round at different points (one temporal step per frame against one non-streaming pass, fp32
# per-token terms summed in fp64 against a float64 log_softmax of the bf16 logits).  Measured on an H100 80GB HBM3
# (700 W): at most 1.8e-7 nats per token (audio 6.5e-8, text 1.8e-7) for this model and corpus; the bound leaves 50x.
TF_TOL = 1e-5


# ------------------------------------------------------------------------------------------------ 3. suspend / resume
def _frames(m, cur, n, active):
    out = []
    m.set_active_streams(active)
    for _ in range(n):
        toks = m.forward_step(cur, use_sampling=False, audio_valid=2048, depth_ring_quirk=False)
        out.append(toks.clone())
        cur = toks[:, :, None]
    return out, cur


def test_suspend_resume_a_forked_row(lm):
    """Row 1 forked from row 0 (a shared full page and a copied partial one) runs 30 frames, is packed with row_segments
    and restored into row 0 of a fresh scope; its next 40 frames (past the ring wrap) equal the uninterrupted run's."""
    P, k, n, B = 70, 30, 40, 3
    seq = CORPUS[1][1][:, :P].to(DEV)
    init = lm._get_initial_token()[0]
    feed = torch.cat([init, seq], 1)

    def start():
        lm.reserve_kv([0], P + k + n)
        lm.prefill_streams({0: feed[:, :-1]})
        lm.fork_kv(0, [1], P + k + n)
        cur = torch.zeros(B, 9, 1, dtype=torch.int64, device=DEV)
        cur[0, :, 0] = cur[1, :, 0] = feed[:, -1]
        return cur

    with lm.streaming(B, kv_pages=12):
        cur = start()
        whole, _ = _frames(lm, cur, k + n, [1, 1, 0])
    with lm.streaming(B, kv_pages=12):
        cur = start()
        _, cur = _frames(lm, cur, k, [1, 1, 0])
        st = lm._state
        regions = st.row_segments(1, P + k)
        table, nbytes = row_state.layout(regions)
        blob = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
        s = torch.cuda.current_stream()
        row_state.run("gather", row_state.pinned_table(table), len(table), blob, s, 16)
        torch.cuda.synchronize()
        last = cur[1, :, 0].clone()
    with lm.streaming(B, kv_pages=12):
        lm.reserve_kv([0], P + k + n)
        st = lm._state
        regions = st.row_segments(0, P + k)
        table, nb = row_state.layout(regions)
        assert nb == nbytes
        row_state.run("scatter", row_state.pinned_table(table), len(table), blob, torch.cuda.current_stream(), 16)
        st.pos_host[0] = P + k
        cur = torch.zeros(B, 9, 1, dtype=torch.int64, device=DEV)
        cur[0, :, 0] = last
        resumed, _ = _frames(lm, cur, n, [1, 0, 0])
    for i in range(n):
        assert torch.equal(resumed[i][0], whole[k + i][1]), i
