"""Paged KV for duplex serving (-m gpu): the paged Kyutai pair-RoPE append against its contiguous form, a paged
`LMGen.streaming` scope against a contiguous one, and both duplex engines on pages against the same engines on contiguous
rings -- with a pool large enough for every session, and with a pool that runs short and evicts.  Paging changes
addresses only, so every comparison is bit for bit."""
import dataclasses
import math

import numpy as np
import pytest
import torch

from oracle import lm_oracle as LO
from oracle import moshi_oracle as MO
from rstnet_b200 import _lib, ops
from rstnet_b200._lib import RstnetError
from rstnet_b200.lm import Sampling

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
BF = torch.bfloat16
F = 1920
PAGE = 16
CANARY = 1234.0
bits = lambda t: t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------------ 1. the kernel
def _pair(paged, qkv, offset, q, kv, rows, B, H, hd, cap, freqs, pt=None, stride=0, log2=0):
    lib, st = _lib.lib(), ops._stream()
    head = (qkv.data_ptr(), offset.data_ptr(), 1, q.data_ptr(), kv.data_ptr(), rows, B, H, hd, cap, freqs.data_ptr())
    if paged:
        _lib.check(lib.rstnet_lm_rope_pair_kv_append_paged_bf16(*head, pt.data_ptr(), stride, log2, st))
    else:
        _lib.check(lib.rstnet_lm_rope_pair_kv_append_bf16(*head, st))


@pytest.mark.parametrize("B,H,hd", [(3, 4, 64), (5, 2, 128), (1, 8, 32), (6, 3, 16)])
@pytest.mark.parametrize("tn", [1, 2])
def test_paged_pair_append_equals_contiguous(B, H, hd, tn):
    """A ring of 200 in pages of 16 (the last page half used), pages shuffled across streams, positions before and past
    the wrap; one stream's current page unmapped: its q_out rows and the pool keep their canaries."""
    g = torch.Generator().manual_seed(B * 100 + H * 10 + hd + tn)
    cap, log2, n_pages = 200, 4, 40 * B
    stride = -(-cap // PAGE)
    offs = torch.tensor([7, 199, 213, 15, 460, 398][:B], dtype=torch.int64)
    offset = offs.to(DEV)
    table = torch.randperm(n_pages, generator=g)[:B * stride].view(stride, B).t().contiguous().to(torch.int32)
    rows = tn * B
    if B > 1:                                      # the last stream's first slot lies on an unmapped page
        table[B - 1, (int(offs[B - 1]) % cap) >> log2] = -1
    pt = table.to(DEV)
    freqs = torch.exp(torch.arange(hd // 2, dtype=torch.float32) * (-math.log(10000.0) * 2 / hd)).to(DEV)
    qkv = torch.randn(rows, 3 * H * hd, generator=g).to(DEV, BF)
    kv_c = torch.randn(2, B, H, cap, hd, generator=g).to(DEV, BF)
    pool = torch.full((n_pages, 2, H, PAGE, hd), CANARY, dtype=BF, device=DEV)
    q_c = torch.full((rows, H * hd), CANARY, dtype=BF, device=DEV)
    q_p = q_c.clone()
    _pair(False, qkv, offset, q_c, kv_c, rows, B, H, hd, cap, freqs)
    _pair(True, qkv, offset, q_p, pool, rows, B, H, hd, cap, freqs, pt, stride, log2)
    torch.cuda.synchronize()
    written = torch.zeros(n_pages, PAGE, dtype=torch.bool)
    for r in range(rows):
        b, tl = r % B, r // B
        slot = (int(offs[b]) + tl) % cap
        page = int(table[b, slot >> log2])
        if page < 0:
            assert bool((q_p[r] == CANARY).all()), r                       # nothing written, q_out included
            continue
        assert torch.equal(bits(q_p[r]), bits(q_c[r])), r
        assert torch.equal(bits(pool[page, :, :, slot & (PAGE - 1)]), bits(kv_c[:, b, :, slot])), r
        written[page, slot & (PAGE - 1)] = True
    assert bool((pool.permute(0, 3, 1, 2, 4)[~written.to(DEV)] == CANARY).all())
    assert written.any()


# ------------------------------------------------------------------------------------------------------ 2. LMGen
MCFG = dataclasses.replace(MO.SMALL, context=40)     # 3 pages of 16 per ring, the last half used


@pytest.fixture(scope="module")
def moshi():
    from rstnet_b200.moshi import LMModel
    m = LMModel(**MCFG.reference_kwargs())
    m.load_state_dict(MO.synthetic_weights(MCFG, seed=5), strict=True)
    return m.to(DEV, BF).eval()


def _grow(model, rows):
    """reserve one more page for each listed row whose next position lies past its pages (the engines' policy)"""
    st = model._paged()
    for r in rows:
        if st.pos_host[r] + 1 > st.pages.limit[r]:
            model.reserve_kv([r], (int(st.pages.held[r]) + 1) * PAGE)


def test_lmgen_paged_equals_contiguous(moshi):
    """Rows admitted at different ticks with their own settings and seeds, held rows, a row restarted; 70 steps over a
    ring of 40 in pages of 16, so every row crosses pages and wraps."""
    from rstnet_b200.moshi import LMGen
    B, T = 4, 70
    n_user = MCFG.n_q - MCFG.dep_q
    admit = {0: [0, 1], 5: [2], 11: [3], 40: [0]}
    held = {(t, 1) for t in range(20, 25)} | {(t, 3) for t in range(30, 33)}
    samplings = [Sampling(top_k=20, temp=0.9), Sampling(use_sampling=False), Sampling(top_p=0.8, top_p_text=0.9), Sampling()]
    inp = torch.randint(0, MCFG.card, (T, B, n_user, 1), generator=torch.Generator().manual_seed(3)).to(DEV)
    runs = []
    for paged in (False, True):
        gen = LMGen(moshi, use_sampling=True, temp=0.8, top_k=250)
        res = []
        with gen.streaming(B, kv_pages=B * 3 if paged else None, kv_page=PAGE):
            live = np.zeros(B, dtype=bool)
            for t in range(T):
                for r in admit.get(t, []):
                    if paged:
                        gen.reserve_kv([r], PAGE)
                    gen.reset_streaming(streams=[r])
                    gen.set_stream_sampling([r], samplings[r], seed=100 + r + t)
                    live[r] = True
                mask = np.array([live[r] and (t, r) not in held for r in range(B)], dtype=np.int64)
                gen.set_active_streams(torch.from_numpy(mask))
                if paged:
                    _grow(moshi, np.flatnonzero(mask))
                out = gen.step(inp[t])
                valid = gen.valid_rows().copy()
                res.append((valid, None if out is None else out[torch.from_numpy(valid).to(DEV)].cpu()))
            if paged:
                assert int(moshi._state.pos_host.max()) > MCFG.context          # the ring wrapped
                assert gen.kv_pages_free == 1        # rows 1-3 hold their whole rings, row 0 (restarted at 40) two pages
                gen.release_kv(range(B))
                assert gen.kv_pages_free == B * 3
                assert gen.kv_page_bytes == MCFG.num_layers * 2 * MCFG.dim * PAGE * 2
        runs.append(res)
    for t, ((va, oa), (vb, ob)) in enumerate(zip(*runs)):
        assert np.array_equal(va, vb), t
        assert (oa is None) == (ob is None), t
        if oa is not None:
            assert torch.equal(oa, ob), t
    assert sum(int(v.sum()) for v, _ in runs[0]) > 150


def test_lmgen_paged_guard(moshi):
    """An active row that would write past its pages raises before any launch, with every counter unchanged; a held row
    without pages steps; a contiguous scope has no page methods."""
    from rstnet_b200.moshi import LMGen
    B = 2
    gen = LMGen(moshi, use_sampling=False)
    inp = torch.zeros(B, MCFG.n_q - MCFG.dep_q, 1, dtype=torch.int64, device=DEV)
    with gen.streaming(B, kv_pages=4, kv_page=PAGE):
        gen.reserve_kv([0], PAGE)
        gen.set_active_streams(torch.tensor([1, 0]))
        for _ in range(PAGE):
            gen.step(inp)
        ms = moshi._state
        snap = (ms.pos_host.copy(), ms.offset.cpu().clone(), gen._st.off_host.copy(), gen._st.off.cpu().clone())
        with pytest.raises(RstnetError):
            gen.step(inp)
        assert np.array_equal(ms.pos_host, snap[0]) and torch.equal(ms.offset.cpu(), snap[1])
        assert np.array_equal(gen._st.off_host, snap[2]) and torch.equal(gen._st.off.cpu(), snap[3])
        gen.reserve_kv([0], 2 * PAGE)
        gen.step(inp)
        assert int(ms.pos_host[0]) == PAGE + 1 and int(ms.pos_host[1]) == 0
        with pytest.raises(RstnetError):
            gen.reserve_kv([1], 1000)                                        # 3 more pages wanted, 2 free
        assert gen.kv_pages_free == 2
    with gen.streaming(B):
        with pytest.raises(RstnetError):
            gen.reserve_kv([0], PAGE)


# ------------------------------------------------------------------------------------------------------ 3. engines
@pytest.fixture(scope="module")
def codec(official_weights):
    from rstnet_b200.codec import MimiCodec
    c = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    c.load_state_dict(official_weights, strict=True)
    c = c.to(DEV).eval()
    c.use_cuda_graphs, c.streaming_tensor_cores = True, True
    yield c
    c._stream_state = None


@pytest.fixture(scope="module")
def gpt():
    from rstnet_b200.lm import GPT, Config
    cfg = dataclasses.replace(LO.SMALL, context=40, block_size=256)
    m = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                   intermediate_size=cfg.intermediate_size, padded_vocab_size=cfg.padded_vocab_size, audio_card=cfg.audio_card,
                   n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim, codecformer_heads=cfg.codecformer_heads,
                   codecformer_layers=cfg.codecformer_layers, codecformer_dim_feedforward=cfg.codecformer_dim_feedforward,
                   context=cfg.context))
    m.load_state_dict(LO.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05), strict=True)
    m.use_cuda_graphs = True
    m = m.to(DEV, BF).eval()
    yield m
    m._state = None


def _engine(kind, codec, gpt, moshi, B, kv_pages):
    from rstnet_b200.moshi import LMGen
    from rstnet_b200.serve import DuplexEngine, MoshiDuplexEngine
    kw = {} if kv_pages is None else dict(kv_pages=kv_pages, kv_page=PAGE)
    if kind == "gpt":
        return DuplexEngine(codec, gpt, B, **kw)
    return MoshiDuplexEngine(codec, LMGen(moshi, use_sampling=True, temp=0.8, top_k=250), B, **kw)


# session: (admission tick, sampling, seed, ticks without audio)
PLAN = {"a": (0, Sampling(top_k=20, temp=0.9), 11, set()), "b": (0, None, 12, {9, 10, 11}),
        "c": (3, Sampling(use_sampling=False), 13, set()), "d": (6, Sampling(top_p=0.8), 14, {20})}
TICKS = 56
AUDIO = {s: 0.1 * torch.randn(F * TICKS, generator=torch.Generator().manual_seed(60 + i)) for i, s in enumerate(PLAN)}


def _serve(engine, kv_headroom=0):
    """-> {session: [(tokens, pcm) per step]}, {tick: [evicted sessions]}"""
    from rstnet_b200.serve import FrameScheduler
    sch = FrameScheduler(engine, engine.B, kv_headroom=kv_headroom)
    got, sent, evicted = {s: [] for s in PLAN}, {s: 0 for s in PLAN}, {}
    for t in range(TICKS):
        for s, (a, sp, seed, _) in PLAN.items():
            if t == a:
                sch.admit(s, sampling=sp, seed=seed)
        for s in sch.sessions():
            if t not in PLAN[s][3]:
                sch.push(s, AUDIO[s][F * sent[s]:F * (sent[s] + 1)])
                sent[s] += 1
        for s, o in sch.tick().items():
            got[s].append(o)
        ev = sch.take_evicted()
        if ev:
            evicted[t] = ev
        assert sch.take_evicted() == []
    for s in list(sch.sessions()):
        sch.release(s)
    return got, evicted


def _predict(n_pages, cap):
    """The host arithmetic of the paging policy: a session holds one page from admission and needs page i + 1 when it
    is about to write position i * PAGE (i * PAGE < cap); each tick the ready sessions grow oldest first, and one that
    finds the pool empty is evicted (its pages return after the tick's growth)."""
    free, held, pos, order, out = n_pages, {}, {}, [], {}
    for t in range(TICKS):
        for s, (a, *_rest) in PLAN.items():
            if t == a:
                free -= 1
                held[s], pos[s] = 1, 0
                order.append(s)
        ready = [s for s in order if t not in PLAN[s][3]]
        gone = []
        for s in ready:
            if pos[s] == held[s] * PAGE and held[s] * PAGE < cap:
                if free == 0:
                    gone.append(s)
                    continue
                free, held[s] = free - 1, held[s] + 1
        for s in gone:
            free += held.pop(s)
            order.remove(s)
        if gone:
            out[t] = gone
        for s in ready:
            if s not in gone:
                pos[s] += 1
    return out


def _same(a, b):
    assert len(a) == len(b)
    for i, ((ta, pa), (tb, pb)) in enumerate(zip(a, b)):
        assert (ta is None) == (tb is None) and (pa is None) == (pb is None), i
        if ta is not None:
            assert torch.equal(ta, tb) and torch.equal(pa, pb), i


@pytest.mark.parametrize("kind", ["gpt", "moshi"])
def test_engine_on_pages(kind, codec, gpt, moshi):
    B, stride = 4, 3
    ref, none = _serve(_engine(kind, codec, gpt, moshi, B, None))
    assert none == {}
    # a pool for every session's whole ring: the same tokens and PCM, nothing evicted, the pool whole again at the end
    eng = _engine(kind, codec, gpt, moshi, B, B * stride)
    got, evicted = _serve(eng)
    assert evicted == {}
    for s in PLAN:
        _same(got[s], ref[s])
        assert any(p is not None for _, p in got[s]), s
    assert eng.kv_pages_free == B * stride
    # a short pool: evictions at the ticks and in the order the host arithmetic predicts; the survivors unchanged
    n = 8
    eng = _engine(kind, codec, gpt, moshi, B, n)
    got, evicted = _serve(eng)
    want = _predict(n, 40)
    assert evicted == want and len(want) >= 2
    gone = {s for v in want.values() for s in v}
    for s in PLAN:
        if s in gone:
            assert len(got[s]) < len(ref[s]), s
            _same(got[s], ref[s][:len(got[s])])
        else:
            _same(got[s], ref[s])
    assert eng.kv_pages_free == n
