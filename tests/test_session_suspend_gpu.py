"""Session suspend / resume (-m gpu): the segment gather / scatter kernel through pinned host memory, and both duplex
engines -- paged and contiguous, 24 kHz and 16 kHz clients -- whose sessions, suspended mid-run and resumed into another
row, another engine instance or another KV layout, produce the tokens and PCM of an uninterrupted run bit for bit."""
import dataclasses

import numpy as np
import pytest
import torch

from oracle import lm_oracle as LO
from oracle import moshi_oracle as MO
from rstnet_b200 import _lib, ops, row_state
from rstnet_b200._lib import RstnetError
from rstnet_b200.lm import Sampling

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
BF = torch.bfloat16
PAGE = 16


# ------------------------------------------------------------------------------------------------------ 1. the kernel
def _roundtrip(table, nbytes, dev_buf, ctas):
    blob = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)
    st = torch.cuda.current_stream()
    tab = row_state.pinned_table(table)
    row_state.run("gather", tab, len(table), blob, st, ctas)
    torch.cuda.synchronize()
    return blob


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("ctas", [1, 7, 132])
def test_gather_scatter_round_trip(seed, ctas):
    """Random segments over one device buffer -- odd sizes, unaligned bases, count 0, 1 and large -- gathered into pinned
    host memory and scattered into a second buffer filled with canaries: the segments' bytes arrive, every other byte
    keeps its canary, and the blob holds each piece where the table says."""
    rng = np.random.default_rng(seed * 10 + ctas)
    N = 1 << 22
    src = torch.randint(0, 256, (N,), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed)).to(DEV)
    dst = torch.full((N,), 0xA5, dtype=torch.uint8, device=DEV)
    taken = np.zeros(N, dtype=bool)
    rows, regions = [], []
    for i in range(60):
        for _ in range(50):
            kind = rng.integers(4)
            nbytes = int(rng.choice([1, 3, 16, 48, 100, 1024, 4096 + 7])) if kind else int(rng.integers(1, 40000))
            count = int(rng.choice([0, 1, 1, 2, 5, 37])) if kind != 3 else int(rng.integers(100, 600))
            stride = nbytes + int(rng.choice([0, 0, 16, 5, 64]))
            span = stride * max(count - 1, 0) + nbytes
            if span >= N // 8:
                continue
            start = int(rng.integers(0, N - span))
            if rng.random() < 0.6:
                start &= ~15
            idx = (start + np.arange(count)[:, None] * stride + np.arange(nbytes)[None, :]).reshape(-1)
            if count and taken[idx].any():
                continue
            taken[idx] = True
            rows.append((start, stride, nbytes, count))
            regions.append((f"s{i}", row_state.segs((src.data_ptr() + start, stride, nbytes, count))))
            break
    table, nbytes = row_state.layout(regions)
    blob = _roundtrip(table, nbytes, src, ctas)
    host = src.cpu().numpy()
    for (start, stride, nb, count), off in zip(rows, table["staging_offset"]):
        want = np.concatenate([host[start + k * stride:start + k * stride + nb] for k in range(count)]) if count else \
            np.zeros(0, np.uint8)
        assert np.array_equal(blob.numpy()[off:off + nb * count], want)
    table2 = table.copy()
    table2["base"] = table["base"] - src.data_ptr() + dst.data_ptr()
    tab = row_state.pinned_table(table2).to(DEV)             # a device table: checked through a copy to the host
    row_state.run("scatter", tab, len(table2), blob, torch.cuda.current_stream(), ctas)
    torch.cuda.synchronize()
    out, mask = dst.cpu().numpy(), torch.from_numpy(taken).numpy()
    assert np.array_equal(out[mask], host[mask])
    assert (out[~mask] == 0xA5).all()
    assert taken.sum() > 100000


def test_bad_arguments_are_error_returns():
    lib, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    buf = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    blob = torch.zeros(4096, dtype=torch.uint8, pin_memory=True)
    good = row_state.layout([("a", row_state.segs((buf.data_ptr(), 64, 64, 2))), ("b", row_state.segs((buf.data_ptr() + 512, 8, 8, 1)))])[0]

    def call(table, n=None, staging=blob.data_ptr(), ctas=4, fn="gather"):
        tab = row_state.pinned_table(table)
        f = lib.rstnet_segments_gather if fn == "gather" else lib.rstnet_segments_scatter
        return f(tab.data_ptr(), len(table) if n is None else n, staging, ctas, st)

    assert call(good) == 0
    bad = [good.copy() for _ in range(5)]
    bad[0]["base"][0] = 0                                    # null base
    bad[1]["count"][1] = -1                                  # count < 0
    bad[2]["staging_offset"][1] = 100                        # inside the first segment's range
    bad[3]["bytes"][0] = -5
    bad[4]["staging_offset"][0] = -16
    for t in bad:
        assert call(t) != 0
    assert call(good, staging=None) != 0
    assert call(good, ctas=0) != 0
    assert call(good, n=-1) != 0
    assert lib.rstnet_segments_gather(None, 2, blob.data_ptr(), 4, st) != 0
    ov = good.copy()
    ov["stride_bytes"][0] = 32                               # pieces of 64 bytes, 32 apart: overlapping destinations
    assert call(ov, fn="scatter") != 0
    assert call(good, n=0) == 0
    dev_bad = row_state.pinned_table(bad[2]).to(DEV)         # the checks hold for a device table too
    assert lib.rstnet_segments_gather(dev_bad.data_ptr(), len(bad[2]), blob.data_ptr(), 4, st) != 0
    dev_good = row_state.pinned_table(good).to(DEV)
    assert lib.rstnet_segments_gather(dev_good.data_ptr(), len(good), blob.data_ptr(), 4, st) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------------ 2. engines
def _codec(weights):
    from rstnet_b200.codec import MimiCodec
    c = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    c.load_state_dict(weights, strict=True)
    c = c.to(DEV).eval()
    c.use_cuda_graphs, c.streaming_tensor_cores = True, True
    return c


def _gpt():
    from rstnet_b200.lm import GPT, Config
    cfg = dataclasses.replace(LO.SMALL, context=40, block_size=256)
    m = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                   intermediate_size=cfg.intermediate_size, padded_vocab_size=cfg.padded_vocab_size, audio_card=cfg.audio_card,
                   n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim, codecformer_heads=cfg.codecformer_heads,
                   codecformer_layers=cfg.codecformer_layers, codecformer_dim_feedforward=cfg.codecformer_dim_feedforward,
                   context=cfg.context))
    m.load_state_dict(LO.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05), strict=True)
    m.use_cuda_graphs = True
    return m.to(DEV, BF).eval()


def _moshi():
    from rstnet_b200.moshi import LMModel
    cfg = dataclasses.replace(MO.SMALL, context=40)
    m = LMModel(**cfg.reference_kwargs())
    m.load_state_dict(MO.synthetic_weights(cfg, seed=5), strict=True)
    return m.to(DEV, BF).eval()


@pytest.fixture(scope="module")
def models(official_weights):
    """two independent sets of models (a second engine instance needs its own streaming scopes)"""
    sets = [dict(codec=_codec(official_weights), gpt=_gpt(), moshi=_moshi()) for _ in range(2)]
    yield sets
    for s in sets:
        s["codec"]._stream_state = None
        s["gpt"]._state = None
        s["moshi"]._state = None


def _engine(kind, ms, B, kv_pages, rate):
    from rstnet_b200.moshi import LMGen
    from rstnet_b200.serve import DuplexEngine, MoshiDuplexEngine
    kw = dict(sample_rate=rate, kv_page=PAGE)
    if kv_pages is not None:
        kw["kv_pages"] = kv_pages
    if kind == "gpt":
        return DuplexEngine(ms["codec"], ms["gpt"], B, **kw)
    return MoshiDuplexEngine(ms["codec"], LMGen(ms["moshi"], use_sampling=True, temp=0.8, top_k=250), B, **kw)


# session: (admission tick, sampling, seed)
PLAN = {"a": (0, Sampling(top_k=20, temp=0.9), 11), "b": (0, None, 12), "c": (3, Sampling(use_sampling=False), 13),
        "d": (6, Sampling(top_p=0.8), 14), "e": (17, None, 15)}
TICKS, B = 48, 5
STRIDE = 3                                           # pages of 16 per ring of 40


def _audio(rate):
    F = rate * 2 // 25
    return F, {s: 0.1 * torch.randn(F * TICKS, generator=torch.Generator().manual_seed(60 + i)) for i, s in enumerate(PLAN)}


def _serve(eng, rate, suspend=(), eng2=None, on_short="evict", kv_headroom=0):
    """Drive a FrameScheduler over TICKS ticks: every live or suspended session pushes one frame per tick.  suspend:
    (session, suspend tick, resume tick) -- resumed into `eng2`'s scheduler when given (a second engine), else into the
    same one.  -> {session: [(tokens, pcm) per step]}, the scheduler"""
    from rstnet_b200.serve import FrameScheduler
    F, audio = _audio(rate)
    sch = FrameScheduler(eng, eng.B, kv_headroom=kv_headroom, on_short=on_short)
    sch2 = FrameScheduler(eng2, eng2.B) if eng2 is not None else None
    got, sent, moved = {s: [] for s in PLAN}, {s: 0 for s in PLAN}, {}
    for t in range(TICKS):
        for s, ts, tr in suspend:
            if t == ts:
                moved[s] = sch.suspend(s)
        for s, (a, sp, seed) in PLAN.items():
            if t == a:
                sch.admit(s, sampling=sp, seed=seed)
        for s, ts, tr in suspend:
            if t == tr:
                if sch2 is None:
                    sch.resume(s)
                else:
                    row = min(sch2._free)
                    sch2._free.remove(row)
                    eng2.resume_rows([row], [sch.__dict__["_suspended"].pop(s)])
                    sch.__dict__["_suspended_at"].pop(s)
                    sch2._row_of[s], sch2._queue[s] = row, sch._queue.pop(s)
        for s in list(sch.sessions()) + sch.suspended() + (list(sch2.sessions()) if sch2 else []):
            q = sch2 if sch2 is not None and s in sch2.sessions() else sch
            q.push(s, audio[s][F * sent[s]:F * (sent[s] + 1)])
            sent[s] += 1
        for q in (sch, sch2) if sch2 is not None else (sch,):
            for s, o in q.tick().items():
                got[s].append(o)
        assert sch.take_evicted() == []
    return got, sch


def _same(a, b, what):
    assert len(a) <= len(b) and len(a) >= 10, what
    for i, ((ta, pa), (tb, pb)) in enumerate(zip(a, b)):
        assert (ta is None) == (tb is None), (what, i)
        if ta is not None:
            assert torch.equal(ta, tb) and torch.equal(pa, pb), (what, i)


_REF = {}


def _reference(kind, ms, rate):
    if (kind, rate) not in _REF:
        _REF[kind, rate] = _serve(_engine(kind, ms, B, None, rate), rate)[0]
    return _REF[kind, rate]


# b past its first page; d inside its warm-up (Moshi max_delay 1); a after its ring of 40 has wrapped (on pages: the whole
# ring, its last page half used)
SUSPEND = (("b", 17, 22), ("d", 7, 9), ("a", 44, 46))


@pytest.mark.parametrize("rate", [24000, 16000])
@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("kind", ["gpt", "moshi"])
def test_suspend_resume_bit_identical(kind, paged, rate, models):
    """b is suspended at tick 17 while the others tick; e is admitted into b's old row at once (on pages: other pages,
    since b's are in flight until its gather completes); b resumes at tick 22 into another row.  Every session's tokens
    and PCM equal the uninterrupted run's, frame for frame (b and d lag by their suspended ticks)."""
    ref = _reference(kind, models[0], rate)
    eng = _engine(kind, models[0], B, B * STRIDE if paged else None, rate)
    got, sch = _serve(eng, rate, SUSPEND)
    for s in PLAN:
        _same(got[s], ref[s], s)
    assert len(got["b"]) == len(ref["b"]) - 5 and sch.lag == {"b": 5, "d": 2, "a": 2}
    if paged:
        for s in list(sch.sessions()):
            sch.release(s)
        torch.cuda.synchronize()
        eng.reclaim()
        assert eng.kv_pages_free == B * STRIDE


@pytest.mark.parametrize("target", ["second", "contiguous"])
@pytest.mark.parametrize("kind", ["gpt", "moshi"])
def test_resume_into_another_engine(kind, target, models):
    """b leaves a paged engine at tick 17 and goes on from tick 22 in a second engine of the same capacity (paged, or
    contiguous rings) on the same device, while a, c, d, e stay in the first."""
    rate = 24000
    ref = _reference(kind, models[0], rate)
    eng = _engine(kind, models[0], B, B * STRIDE, rate)
    eng2 = _engine(kind, models[1], B, B * STRIDE if target == "second" else None, rate)
    got, _ = _serve(eng, rate, (("b", 17, 22),), eng2=eng2)
    for s in PLAN:
        _same(got[s], ref[s], s)


@pytest.mark.parametrize("kind", ["gpt", "moshi"])
def test_incompatible_engine_raises(kind, models):
    eng = _engine(kind, models[0], B, B * STRIDE, 24000)
    eng.reset_rows([0], seed=3)
    st = eng.suspend_rows([0])[0]
    torch.cuda.synchronize()
    other = _engine(kind, models[1], B, B * STRIDE, 16000)            # another client rate
    with pytest.raises(RstnetError):
        other.resume_rows([0], [st])
    assert other.kv_pages_free == B * STRIDE
    with pytest.raises(RstnetError):
        _engine("moshi" if kind == "gpt" else "gpt", models[1], B, None, 24000).resume_rows([0], [st])
    assert st.nbytes > 0 and st.positions == 0


@pytest.mark.parametrize("kind", ["gpt", "moshi"])
def test_scheduler_suspends_instead_of_evicting(kind, models):
    """A pool of 8 pages for 5 sessions of up to 3 pages: with on_short="suspend" nobody is evicted, sessions are
    suspended and resumed, and each one's outputs equal its uninterrupted run."""
    rate = 24000
    ref = _reference(kind, models[0], rate)
    eng = _engine(kind, models[0], B, 8, rate)
    got, sch = _serve(eng, rate, on_short="suspend")
    assert sch.suspensions > 0 and sch.resumes > 0
    for s in PLAN:
        if s not in sch.suspended():
            _same(got[s], ref[s], s)


def _script(eng, actions, ticks, seeds):
    """Drive a FrameScheduler: actions {tick: [(verb, session)]} run before the tick's pushes (verbs: admit, release,
    suspend, resume, sync = wait for the session's gather and reclaim its pages, or a callable(sch, eng)).  Every live
    or suspended session pushes one frame per tick.  -> {session: [(tokens, pcm) per step]}"""
    from rstnet_b200.serve import FrameScheduler
    F, audio = _audio(24000)
    sch = FrameScheduler(eng, eng.B)
    got, sent, states = {s: [] for s in seeds}, {s: 0 for s in seeds}, {}
    for t in range(ticks):
        for verb, s in actions.get(t, []):
            if callable(verb):
                verb(sch, eng, states)
            elif verb == "admit":
                sch.admit(s, seed=seeds[s])
            elif verb == "release":
                sch.release(s)
            elif verb == "suspend":
                states[s] = sch.suspend(s)
            elif verb == "resume":
                sch.resume(s)
            elif verb == "sync":
                states[s].ready.synchronize()
                eng.reclaim()
        for s in list(sch.sessions()) + sch.suspended():
            sch.push(s, audio["abcde"[list(seeds).index(s)]][F * sent[s]:F * (sent[s] + 1)])
            sent[s] += 1
        for s, o in sch.tick().items():
            got[s].append(o)
        assert sch.take_evicted() == []
    return got


@pytest.mark.parametrize("kind", ["gpt", "moshi"])
def test_ordering_of_freed_pages_and_rows(kind, models):
    """A pool of 6 pages of 16, 3 rows.  t 20: A (2 pages) is suspended; its pages stay out of the pool until its gather
    has completed, then C is admitted into A's row and takes A's pages and writes them for 10 ticks before A resumes into
    row 2 (reserving to its page boundary).  t 34: X is suspended, resumed into its old row, released and B admitted into
    that row at once, before any tick: B's restart waits for X's scatter.  Every session equals its run in a contiguous
    engine without suspensions."""
    seeds = {"A": 21, "X": 22, "C": 23, "B": 24}
    T = 46
    ref = _script(_engine(kind, models[0], 3, None, 24000),
                  {0: [("admit", "A"), ("admit", "X")], 20: [("admit", "C")], 34: [("release", "X"), ("admit", "B")]}, T, seeds)
    seen = {}

    def before_a(sch, eng, states):
        seen["a_pages"] = set(eng._kv_lm._paged().pages.table[0, :2].tolist())
        seen["free"] = eng.kv_pages_free

    def after_a(sch, eng, states):
        assert eng.kv_pages_free == seen["free"] == 2          # A's pages are in flight, not free

    def c_took_a(sch, eng, states):
        pages = eng._kv_lm._paged().pages
        assert sch.sessions()["C"] == 0 and int(pages.table[0, 0]) in seen["a_pages"]

    def a_back(sch, eng, states):
        pages = eng._kv_lm._paged().pages
        assert sch.sessions()["A"] == 2 and pages.held[2] == 2 and pages.limit[2] == 32

    def x_full(sch, eng, states):
        assert eng.kv_pages_free == 0                          # X's 3 pages in flight, the pool otherwise full

    eng = _engine(kind, models[0], 3, 6, 24000)
    got = _script(eng, {0: [("admit", "A"), ("admit", "X")],
                        20: [(before_a, None), ("suspend", "A"), (after_a, None), ("sync", "A"), ("admit", "C"), (c_took_a, None)],
                        30: [("resume", "A"), (a_back, None)],
                        34: [("suspend", "X"), (x_full, None), ("sync", "X"), ("resume", "X"), ("release", "X"), ("admit", "B")]},
                  T, seeds)
    for s in seeds:
        _same(got[s], ref[s], s)
    assert len(got["A"]) == len(ref["A"]) - 10 and len(got["B"]) == len(ref["B"]) == T - 34
