"""GPU tests (-m gpu) of serving the Moshi-style LMGen to a batch of sessions: the per-row delay-cache kernels
(csrc/delay_cache.cu) against a restatement of LMGen.step's cache arithmetic, per-row admission / hold / state round-trip
of `LMGen`, decisions against the oracle per row, and `MoshiDuplexEngine` under `FrameScheduler`.  Greedy decoding."""
import pytest
import torch

from oracle import moshi_oracle as M
from rstnet_b200 import _lib, ops
from rstnet_b200.moshi import LMGen, LMModel

pytestmark = pytest.mark.gpu
DEV, BF = "cuda", torch.bfloat16
CFG = M.SMALL
N_USER = CFG.n_q - CFG.dep_q


@pytest.fixture(scope="module")
def moshi():
    w = M.synthetic_weights(CFG, seed=5)
    m = LMModel(**CFG.reference_kwargs())
    m.load_state_dict(w, strict=True)
    return m.to(DEV, BF).eval(), w


def _inputs(T, B, seed):
    return torch.randint(0, CFG.card, (T, B, N_USER, 1), generator=torch.Generator().manual_seed(seed))


# ------------------------------------------------------------------------------------------- kernels vs restatement
def _ref_cache_in(cache, off, active, delays, user, dep_q, text_init, audio_init):
    """LMGenOracle.step's writes before the LM, row by row with the row's own offset; held rows only read."""
    cache = cache.clone()
    B, K, CT = cache.shape
    seq = torch.empty(B, K, dtype=torch.int64)
    for b in range(B):
        o = int(off[b])
        if active[b]:
            for q in range(K - dep_q - 1):
                k = dep_q + 1 + q
                cache[b, k, (o + delays[k]) % CT] = user[b, q]
            for k, d in enumerate(delays):
                if o <= d:
                    cache[b, k, o % CT] = text_init if k == 0 else audio_init
            seq[b] = cache[b, :, o % CT]
        else:
            seq[b] = cache[b, :, o % CT].clamp(min=-1)
    return cache, seq


def _ref_cache_out(cache, off, valid, out, active, delays, tokens, dep_q, max_delay):
    """LMGenOracle.step's write-back, offset advance and gather, row by row; held rows untouched."""
    cache, off, valid, out = cache.clone(), off.clone(), valid.clone(), out.clone()
    CT = cache.shape[2]
    gd = torch.tensor(delays[:dep_q + 1])
    for b in range(cache.shape[0]):
        if not active[b]:
            continue
        off[b] += 1
        o = int(off[b])
        cache[b, :dep_q + 1, o % CT] = tokens[b]
        out[b] = cache[b, torch.arange(dep_q + 1), (o - max_delay + gd) % CT]
        valid[b] = int(o > max_delay)
    return cache, off, valid, out


SYNTH_DELAYS = (0, 0, 1, 3, 2, 0, 1, 3, 2, 0, 3, 1, 2, 0, 3, 1, 2)     # max 3: CT = 5


@pytest.mark.parametrize("delays,B,seed", [(CFG.delays, 37, 1), (CFG.delays, 256, 2), (SYNTH_DELAYS, 37, 3),
                                           (SYNTH_DELAYS, 200, 4)])
def test_delay_cache_kernels_vs_restatement(delays, B, seed):
    L = _lib.lib()
    g = torch.Generator().manual_seed(seed)
    K, dep_q, max_delay = len(delays), CFG.dep_q, max(delays)
    CT = max_delay + 2
    text_init, audio_init = CFG.text_card, CFG.card
    ids = lambda *shape: torch.randint(-2, CFG.card + 1, shape, generator=g)     # incl. -2 ungenerated, -1 zero, init
    for trial in range(4):
        cache = ids(B, K, CT)
        off = torch.randint(0, 3 * CT, (B,), generator=g)
        off[:2 * CT] = torch.arange(2 * CT)                          # every offset around the delays
        active = (torch.rand(B, generator=g) < 0.7).long()
        user = ids(B, K - dep_q - 1)
        tokens = ids(B, dep_q + 1)
        valid = (off > max_delay).long()
        out = torch.full((B, dep_q + 1), 7777, dtype=torch.int64)
        d = {n: t.to(DEV) for n, t in dict(cache=cache, off=off, active=active, user=user, tokens=tokens, valid=valid,
                                          out=out).items()}
        d["delays"] = torch.tensor(delays, dtype=torch.int64, device=DEV)
        d["seq"] = torch.full((B, K + 3), 5555, dtype=torch.int64, device=DEV)          # row stride K + 3: padding untouched
        st = ops._stream()
        _lib.check(L.rstnet_lm_delay_cache_in(d["cache"].data_ptr(), d["off"].data_ptr(), d["active"].data_ptr(),
                                              d["delays"].data_ptr(), d["user"].data_ptr(), K - dep_q - 1, d["seq"].data_ptr(),
                                              K + 3, B, K, dep_q, CT, text_init, audio_init, st), "cache_in")
        r_cache, r_seq = _ref_cache_in(cache, off, active, delays, user, dep_q, text_init, audio_init)
        assert torch.equal(d["cache"].cpu(), r_cache), trial
        assert torch.equal(d["seq"][:, :K].cpu(), r_seq), trial
        assert bool((d["seq"][:, K:] == 5555).all())
        _lib.check(L.rstnet_lm_delay_cache_out(d["cache"].data_ptr(), d["off"].data_ptr(), d["active"].data_ptr(),
                                               d["delays"].data_ptr(), d["tokens"].data_ptr(), dep_q + 1, d["out"].data_ptr(),
                                               dep_q + 1, d["valid"].data_ptr(), B, K, dep_q, CT, max_delay, st), "cache_out")
        r_cache, r_off, r_valid, r_out = _ref_cache_out(r_cache, off, valid, out, active, delays, tokens, dep_q, max_delay)
        assert torch.equal(d["cache"].cpu(), r_cache), trial
        assert torch.equal(d["off"].cpu(), r_off) and torch.equal(d["valid"].cpu(), r_valid), trial
        assert torch.equal(d["out"].cpu(), r_out), trial
        held = active == 0
        assert torch.equal(d["cache"].cpu()[held], cache[held]) and bool((d["out"].cpu()[held] == 7777).all())


def test_delay_cache_rejects_bad_shapes():
    L = _lib.lib()
    t = torch.zeros(64, dtype=torch.int64, device=DEV)
    p = t.data_ptr()
    assert L.rstnet_lm_delay_cache_out(p, p, None, p, p, 9, p, 9, p, 2, 17, 8, 4, 1, ops._stream()) != 0   # CT != max_delay + 2
    assert L.rstnet_lm_delay_cache_in(p, p, None, p, p, 8, p, 17, 2, 17, 17, 3, 1, 1, ops._stream()) != 0  # dep_q >= K


# ------------------------------------------------------------------------------------------- LMGen, per row
def _record(gen, o):
    return (None if o is None else o.cpu(), gen.valid_rows().copy(), gen.lm_model._st().active_host.copy())


def _run(m, B, schedule, feed, T):
    """Run an LMGen scope of B rows for T steps.  schedule(t) -> (rows to reset before step t, active mask or None);
    feed(t) -> input [B, 8, 1].  Returns per step: (output or None, valid_rows, active flags)."""
    gen = LMGen(m, use_sampling=False)
    res = []
    with gen.streaming(B):
        for t in range(T):
            reset, mask = schedule(t)
            if reset:
                gen.reset_streaming(streams=reset)
            gen.set_active_streams(mask)
            res.append(_record(gen, gen.step(feed(t).to(DEV))))
    return res


def _row_outputs(res, r, since=0):
    """Row r's results at the steps it took from step `since` on: (valid, tokens if valid)."""
    return [(bool(v[r]), o[r].clone() if v[r] else None) for o, v, act in res[since:] if act[r]]


def _same(a, b):
    assert len(a) == len(b)
    for i, ((va, ta), (vb, tb)) in enumerate(zip(a, b)):
        assert va == vb, i
        if va:
            assert torch.equal(ta, tb), i


def test_lmgen_all_rows_together_is_reference_behaviour(moshi):
    m, _ = moshi
    B, x = 3, _inputs(6, 3, 11)
    gen = LMGen(m, use_sampling=False)
    md = max(CFG.delays)
    with gen.streaming(B):
        for t in range(6):
            o = gen.step(x[t].to(DEV))
            assert (o is None) == (t < md)
            assert list(gen.valid_rows()) == [t >= md] * B and gen._st.offset == t + 1


def test_lmgen_step_is_one_graph_replay(moshi, monkeypatch):
    """After the warm-up calls, a step is one input copy, one graph replay and the result copy: no library launch from the
    host and no eager cache arithmetic."""
    m, _ = moshi
    B, x = 4, _inputs(6, 4, 12)
    gen = LMGen(m, use_sampling=False)
    with gen.streaming(B):
        for t in range(3):
            gen.step(x[t].to(DEV))
        torch.cuda.synchronize()
        n = [0]
        orig = torch.cuda.CUDAGraph.replay

        def counted(self):
            n[0] += 1
            return orig(self)
        monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", counted)
        inp = x[3].to(DEV)
        l0 = _lib.launch_count()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            gen.step(inp)
            torch.cuda.synchronize()
        assert n[0] == 1 and _lib.launch_count() == l0
        names = [e.name for e in prof.events()]
        graph = sum(nm == "cudaGraphLaunch" for nm in names)
        eager = sum(nm.startswith("cudaLaunchKernel") for nm in names)
        print(f"LMGen.step: {graph} graph launch(es), {eager} eager kernel launch(es)")
        assert graph == 1 and eager <= 2


def test_lmgen_admission(moshi):
    """B = 4, 6 steps, reset row 2, 8 more: row 2 equals a fresh scope fed row 2's inputs from the reset (tokens, valid
    pattern, None warm-up); the other rows equal an uninterrupted run."""
    m, _ = moshi
    B, T = 4, 14
    x = _inputs(T, B, 13)
    live = _run(m, B, lambda t: ([2] if t == 6 else [], None), lambda t: x[t], T)
    plain = _run(m, B, lambda t: ([], None), lambda t: x[t], T)
    fresh = _run(m, B, lambda t: ([], None), lambda t: x[6 + t], T - 6)
    for r in (0, 1, 3):
        _same(_row_outputs(live, r), _row_outputs(plain, r))
    _same(_row_outputs(live, 2, since=6), _row_outputs(fresh, 2))
    assert [o is None for o, _, _ in fresh] == [t < max(CFG.delays) for t in range(T - 6)]
    assert [bool(v[2]) for _, v, _ in live[6:]] == [o is not None for o, _, _ in fresh]


def test_lmgen_hold(moshi):
    """Row 1 held for 3 steps mid-stream and row 3 held for its first 2 steps: each equals a run in which those steps
    never happened for it; a held row's cache, offset and valid flag do not change."""
    m, _ = moshi
    B, T = 4, 12
    held = {1: {4, 5, 6}, 3: {0, 1}}
    real = _inputs(T, B, 14)                                   # real[j, r]: row r's j-th real input
    junk = _inputs(T, B, 15)
    count = {r: 0 for r in range(B)}
    feeds = []
    for t in range(T):
        f = junk[t].clone()
        for r in range(B):
            if t not in held.get(r, ()):
                f[r] = real[count[r], r]
                count[r] += 1
        feeds.append(f)
    mask = lambda t: [0 if t in held.get(r, ()) else 1 for r in range(B)]
    gen = LMGen(m, use_sampling=False)
    res = []
    with gen.streaming(B):
        for t in range(T):
            gen.set_active_streams(mask(t))
            before = {r: (gen._st.cache[r].clone(), int(gen._st.off[r]), int(gen._st.valid[r]))
                      for r in range(B) if not mask(t)[r]}
            o = gen.step(feeds[t].to(DEV))
            for r, (c, off, v) in before.items():
                assert torch.equal(gen._st.cache[r], c) and int(gen._st.off[r]) == off and int(gen._st.valid[r]) == v, (t, r)
                assert not gen.valid_rows()[r]
            res.append(_record(gen, o))
    ref = _run(m, B, lambda t: ([], None), lambda t: real[t], T)
    for r in range(B):
        mine = _row_outputs(res, r)
        _same(mine, _row_outputs(ref, r)[:len(mine)])


def test_lmgen_rows_admitted_at_different_ticks_vs_oracle(moshi):
    """Each row, from its admission, makes the oracle's argmax (the oracle teacher-forced with our tokens, one oracle
    scope per row), as test_lmgen_step_closed_loop checks for a scope started at once."""
    m, w = moshi
    B, T = 3, 12
    admit = {0: 0, 1: 3, 2: 5}
    x = _inputs(T, B, 16)
    gen = LMGen(m, use_sampling=False)
    wb = {k: v.to(BF) for k, v in w.items()}
    ora = {}
    stats = {r: [0, 0, 0.0] for r in range(B)}
    with gen.streaming(B), torch.no_grad():
        for t in range(T):
            new = [r for r, a in admit.items() if a == t]
            if new:
                gen.reset_streaming(streams=new)
                for r in new:
                    ora[r] = M.LMGenOracle(wb, CFG, 1)
            gen.step(x[t].to(DEV))
            CT = gen._st.cache.shape[2]
            for r, o in ora.items():
                pos = int(gen._st.off_host[r]) % CT
                ours = gen._st.cache[r:r + 1, :CFG.dep_q + 1, pos].cpu()
                o.step(x[t][r:r + 1], force=ours)
                _, _, text_logits, alog = o.last
                lt = text_logits.float()[:, 0, 0]
                d = torch.cat([lt.max(-1).values - lt.gather(1, ours[:, :1])[:, 0],
                               (alog.float().max(-1).values - alog.float().gather(2, ours[:, 1:, None])[:, :, 0]).flatten()])
                stats[r][0] += int((d == 0).sum()); stats[r][1] += d.numel(); stats[r][2] = max(stats[r][2], float(d.max()))
    for r, (exact, n, worst) in stats.items():
        print(f"row {r} (admitted at tick {admit[r]}): {exact}/{n} decisions are the oracle's exact argmax; worst deficit {worst:.3f}")
        assert worst <= 0.1 and exact >= 0.8 * n


def test_lmgen_streaming_state_round_trip(moshi):
    m, _ = moshi
    B, T = 3, 10
    x, y = _inputs(T, B, 17), _inputs(4, B, 18)
    plain = _run(m, B, lambda t: ([1] if t == 2 else [], [1, 0, 1] if t == 3 else None), lambda t: x[t], T)
    gen = LMGen(m, use_sampling=False)
    res = []

    def one(t):
        if t == 2:
            gen.reset_streaming(streams=[1])
        gen.set_active_streams([1, 0, 1] if t == 3 else None)
        res.append(_record(gen, gen.step(x[t].to(DEV))))

    gen.streaming_forever(B)
    for t in range(5):
        one(t)
    parked = gen.get_streaming_state()
    gen.streaming_forever(B)                                       # another scope runs in between
    for t in range(4):
        gen.step(y[t].to(DEV))
    gen.set_streaming_state(parked)
    for t in range(5, T):
        one(t)
    for r in range(B):
        _same(_row_outputs(res, r), _row_outputs(plain, r))
    other = LMGen(m, use_sampling=False)
    with pytest.raises(RuntimeError):
        other.set_streaming_state(parked)
    gen.set_streaming_state({"": None})
    assert not gen.is_streaming


# ------------------------------------------------------------------------------------------- the engine
@pytest.fixture(scope="module")
def codec(official_weights):
    from rstnet_b200.codec import MimiCodec
    c = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    c.load_state_dict(official_weights, strict=True)
    c = c.to(DEV).eval()
    c.use_cuda_graphs, c.streaming_tensor_cores = True, True
    return c


def _audio(n, L, seed):
    g = torch.Generator().manual_seed(seed)
    return 0.1 * torch.randn(n, L, generator=g)


def test_moshi_engine_sessions_vs_hand_loop(moshi, codec):
    """Sessions admitted at different ticks, one with gaps in its audio: no PCM for exactly the first max_delay ticks of
    each, then (tokens, PCM) equal to the reference loop (encode -> step -> decode, decode skipped while step returns
    None) at the same B in which the session ran alone from its admission."""
    from rstnet_b200.serve import FrameScheduler, MoshiDuplexEngine
    m, _ = moshi
    B, ticks = 3, 9
    plan = {"a": (0, set()), "b": (2, set()), "c": (1, {4, 5})}       # session: (admission tick, ticks without audio)
    audio = {s: _audio(1, 1920 * ticks, 20 + i)[0] for i, s in enumerate(plan)}
    eng = MoshiDuplexEngine(codec, LMGen(m, use_sampling=False), B)
    sch = FrameScheduler(eng, B)
    got = {s: [] for s in plan}
    nxt = {s: 0 for s in plan}
    rows = {}
    for t in range(ticks):
        for s, (a, gaps) in plan.items():
            if t == a:
                rows[s] = sch.admit(s)
            if t >= a and t not in gaps:
                sch.push(s, audio[s][1920 * nxt[s]:1920 * (nxt[s] + 1)])
                nxt[s] += 1
        for s, v in sch.tick().items():
            got[s].append(v)
    md = max(CFG.delays)
    for s in plan:
        n = len(got[s])
        assert [p is None for _, p in got[s]] == [i < md for i in range(n)], s
        gen = LMGen(m, use_sampling=False)
        r = rows[s]
        with codec.streaming(B), gen.streaming(B):
            for i in range(n):
                pcm = audio[s][1920 * i:1920 * (i + 1)].reshape(1, 1, -1).expand(B, 1, -1).contiguous().to(DEV)
                toks = gen.step(codec.encode(pcm))
                if toks is None:
                    assert got[s][i] == (None, None)
                    continue
                out = codec.decode(toks[:, 1:]).cpu()
                tk, p = got[s][i]
                assert torch.equal(tk, toks[r, :, 0].cpu()), (s, i)
                assert torch.equal(p, out[r, 0]), (s, i)
    codec._stream_state = None


def test_moshi_engine_16k(moshi, codec):
    from rstnet_b200.serve import MoshiDuplexEngine
    m, _ = moshi
    B, F = 2, int(0.08 * 16000)
    eng = MoshiDuplexEngine(codec, LMGen(m, use_sampling=False), B, sample_rate=16000)
    x = _audio(B, 4 * F, 30)
    for i in range(4):
        out = eng.step({r: x[r, i * F:(i + 1) * F] for r in range(B)}, list(range(B)))
        for r in range(B):
            tk, p = out[r]
            if i < max(CFG.delays):
                assert tk is None and p is None
            else:
                assert tk.shape == (CFG.dep_q + 1,) and p.shape == (F,) and bool(torch.isfinite(p).all())
    codec._stream_state = None


def test_moshi_engine_rejects_mismatched_codec(moshi):
    from rstnet_b200._lib import RstnetError
    from rstnet_b200.codec import MimiCodec
    from rstnet_b200.serve import MoshiDuplexEngine
    m, _ = moshi
    c = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=4)
    with pytest.raises(RstnetError):
        MoshiDuplexEngine(c, LMGen(m), 2)
    with pytest.raises(RstnetError):
        MoshiDuplexEngine(c, LMGen(m), 257)
