"""GPU tests (-m gpu) of prompted Moshi generation: the delay-cache prompt kernel against P launches of cache_in /
cache_out, the paged row-map pair-RoPE against the contiguous row-map form, prompted LMGen rows against the oracle forced
through the prompt, self-consistency with stepped rows, the exact invariants of LMGen.prefill_streams and generate_many,
prompted sessions in MoshiDuplexEngine / FrameScheduler, and `offline continue`."""
import dataclasses
import json

import numpy as np
import pytest
import torch

from oracle import moshi_oracle as M
from rstnet_b200 import _lib, ops
from rstnet_b200.lm import Sampling, row_chunk_positions
from rstnet_b200.moshi import LMGen, LMModel, generate_many, prompt_from_aligned

pytestmark = pytest.mark.gpu
DEV, BF = "cuda", torch.bfloat16
CFG = dataclasses.replace(M.SMALL, delays=(0, 0, 1, 2, 1, 0, 1, 2, 1, 0, 1, 2, 1, 0, 1, 2, 1))   # max_delay 2: CT = 4
K, DQ = CFG.n_q + 1, CFG.dep_q
N_USER = K - DQ - 1
MD = max(CFG.delays)


@pytest.fixture(scope="module")
def moshi():
    w = M.synthetic_weights(CFG, seed=5)
    m = LMModel(**CFG.reference_kwargs())
    m.load_state_dict(w, strict=True)
    return m.to(DEV, BF).eval(), w


def _seq(L, seed):
    """aligned dialogue codes [K, L]: text ids, then audio ids"""
    g = torch.Generator().manual_seed(seed)
    s = torch.randint(0, CFG.card, (K, L), generator=g)
    s[0] = torch.randint(0, CFG.text_card, (L,), generator=g)
    return s


# ------------------------------------------------------------------------------------------- the prompt kernel
@pytest.mark.parametrize("delays", [CFG.delays, (0,) * K, (0, 3, 1, 0, 2, 3, 1, 0, 2, 0, 3, 1, 2, 0, 3, 1, 2)])
def test_delay_cache_prompt_equals_stepwise_launches(delays):
    L = _lib.lib()
    st = ops._stream()
    B, md = 9, max(delays)
    CT = md + 2
    g = torch.Generator().manual_seed(len(set(delays)))
    lens = {1: 0, 3: 1, 4: md, 5: md + 1, 0: 3 * CT + 5, 7: 40}       # rows 2, 6, 8 are left out
    rows = list(lens)
    cache0 = torch.randint(-2, 50, (B, K, CT), generator=g)
    off0 = torch.randint(0, 7, (B,), generator=g)
    off0[[3, 7]] = 0
    prompts = {r: torch.randint(-2, 50, (K, n), generator=g) for r, n in lens.items()}
    dv = torch.tensor(delays, dtype=torch.int64, device=DEV)
    # P launch pairs per row, rows alone (the others held)
    ref = dict(cache=cache0.clone().to(DEV), off=off0.clone().to(DEV), valid=torch.zeros(B, dtype=torch.int64, device=DEV))
    ref_feed = {}
    seq = torch.zeros(B, K, dtype=torch.int64, device=DEV)
    out = torch.zeros(B, DQ + 1, dtype=torch.int64, device=DEV)
    for r, p in prompts.items():
        act = torch.zeros(B, dtype=torch.int64, device=DEV)
        act[r] = 1
        feeds = []
        for t in range(p.shape[1]):
            user = torch.zeros(B, N_USER, dtype=torch.int64, device=DEV)
            user[r] = p[DQ + 1:, t].to(DEV)
            tok = torch.zeros(B, DQ + 1, dtype=torch.int64, device=DEV)
            tok[r] = p[:DQ + 1, t].to(DEV)
            _lib.check(L.rstnet_lm_delay_cache_in(ref["cache"].data_ptr(), ref["off"].data_ptr(), act.data_ptr(), dv.data_ptr(),
                                                  user.data_ptr(), N_USER, seq.data_ptr(), K, B, K, DQ, CT, CFG.text_card,
                                                  CFG.card, st))
            feeds.append(seq[r].clone())
            _lib.check(L.rstnet_lm_delay_cache_out(ref["cache"].data_ptr(), ref["off"].data_ptr(), act.data_ptr(), dv.data_ptr(),
                                                   tok.data_ptr(), DQ + 1, out.data_ptr(), DQ + 1, ref["valid"].data_ptr(), B, K,
                                                   DQ, CT, md, st))
        ref_feed[r] = torch.stack(feeds) if feeds else torch.zeros(0, K, dtype=torch.int64, device=DEV)
    # one launch, rows in another order, packed with a stride
    order = [7, 1, 4, 0, 5, 3]
    starts = np.concatenate([[0], np.cumsum([lens[r] for r in order])[:-1]]).astype(np.int32)
    total = sum(lens.values())
    packed = torch.full((total, K + 2), 9999, dtype=torch.int64)
    for r, s0 in zip(order, starts):
        packed[s0:s0 + lens[r], :K] = prompts[r].t()
    packed = packed.to(DEV)
    feed = torch.full((total, K + 1), 8888, dtype=torch.int64, device=DEV)
    cache, off = cache0.clone().to(DEV), off0.clone().to(DEV)
    valid = torch.full((B,), 7, dtype=torch.int64, device=DEV)
    r32, l32 = np.array(order, dtype=np.int32), np.array([lens[r] for r in order], dtype=np.int32)
    _lib.check(L.rstnet_lm_delay_cache_prompt(cache.data_ptr(), off.data_ptr(), valid.data_ptr(), dv.data_ptr(), packed.data_ptr(),
                                              K + 2, feed.data_ptr(), K + 1, r32.ctypes.data, starts.ctypes.data, l32.ctypes.data,
                                              len(order), B, K, DQ, CT, md, CFG.text_card, CFG.card, st))
    for r, s0 in zip(order, starts):
        assert torch.equal(feed[s0:s0 + lens[r], :K], ref_feed[r]), r
    assert bool((feed[:, K] == 8888).all())
    moved = [r for r in rows if lens[r] > 0]
    assert torch.equal(cache[moved], ref["cache"][moved]) and torch.equal(off[moved], ref["off"][moved])
    assert torch.equal(valid[moved], ref["valid"][moved])
    still = [r for r in range(B) if r not in moved]                     # P = 0 and rows not listed: untouched
    assert torch.equal(cache[still].cpu(), cache0[still]) and torch.equal(off[still].cpu(), off0[still])
    assert bool((valid[still] == 7).all())
    # bad arguments: an error return, nothing launched, nothing written
    n0 = _lib.launch_count()
    bad = np.array([7, 7], dtype=np.int32)
    assert L.rstnet_lm_delay_cache_prompt(cache.data_ptr(), off.data_ptr(), valid.data_ptr(), dv.data_ptr(), packed.data_ptr(), K + 2,
                                          feed.data_ptr(), K + 1, bad.ctypes.data, starts.ctypes.data, l32.ctypes.data, 2, B, K,
                                          DQ, CT, md, CFG.text_card, CFG.card, st) != 0
    assert _lib.launch_count() == n0 and torch.equal(off[moved], ref["off"][moved])


# ------------------------------------------------------------------------------------------- paged row-map pair-RoPE
def test_paged_rows_pair_rope_equals_contiguous_rows():
    L = _lib.lib()
    st = ops._stream()
    B, H, hd, cap, P = 3, 4, 64, 48, 16
    g = torch.Generator().manual_seed(11)
    # stream 0 crosses a page boundary, stream 1 wraps the ring, stream 2 starts at 0; padding rows in between
    offset = torch.tensor([10, 40, 0], dtype=torch.int64, device=DEV)
    rs = [0] * 12 + [-1] * 3 + [1] * 15 + [2] * 5 + [-1]
    rt = list(range(12)) + [0] * 3 + list(range(15)) + list(range(5)) + [0]
    M_ = len(rs)
    qkv = torch.randn(M_, 3 * H * hd, generator=g).to(DEV, BF)
    freqs = torch.exp(torch.arange(hd // 2, dtype=torch.float32) * (-np.log(10000.0) * 2 / hd)).to(DEV)
    row_s, row_t = (torch.tensor(v, dtype=torch.int32, device=DEV) for v in (rs, rt))
    q_c, q_p = (torch.full((M_, H * hd), 7.0, dtype=BF, device=DEV) for _ in range(2))
    kv_c = torch.full((2, B, H, cap, hd), 5.0, dtype=BF, device=DEV)
    _lib.check(L.rstnet_lm_rope_pair_kv_append_rows_bf16(qkv.data_ptr(), offset.data_ptr(), row_s.data_ptr(), row_t.data_ptr(),
                                                         q_c.data_ptr(), kv_c.data_ptr(), M_, B, H, hd, cap, freqs.data_ptr(), st))
    npg = cap // P
    table = torch.randperm(B * npg, generator=torch.Generator().manual_seed(2)).view(B, npg).to(torch.int32)
    pool = torch.full((B * npg, 2, H, P, hd), 5.0, dtype=BF, device=DEV)
    _lib.check(L.rstnet_lm_rope_pair_kv_append_paged_rows_bf16(qkv.data_ptr(), offset.data_ptr(), row_s.data_ptr(), row_t.data_ptr(),
                                                               q_p.data_ptr(), pool.data_ptr(), M_, B, H, hd, cap, freqs.data_ptr(),
                                                               table.to(DEV).data_ptr(), npg, 4, st))
    assert torch.equal(q_p.view(torch.int16), q_c.view(torch.int16))
    pad = torch.tensor([s < 0 for s in rs], device=DEV)
    assert bool((q_p[pad] == 7.0).all())
    # the pool seen through the table is the contiguous rings, byte for byte (untouched slots included)
    gathered = pool[table.long().to(DEV)]                      # [B, npg, 2, H, P, hd]
    rings = gathered.permute(2, 0, 3, 1, 4, 5).reshape(2, B, H, cap, hd)
    assert torch.equal(rings.view(torch.int16), kv_c.view(torch.int16))
    assert bool((kv_c[:, 1, :, 7:40] == 5.0).all())            # stream 1 wrote slots 40..47 and 0..6 only


# ------------------------------------------------------------------------------------------- against the oracle
def _margin(o, ours):
    _, _, text_logits, alog = o.last
    lt = text_logits.float()[:, 0, 0]
    return torch.cat([lt.max(-1).values - lt.gather(1, ours[:, :1])[:, 0],
                      (alog.float().max(-1).values - alog.float().gather(2, ours[:, 1:, None])[:, :, 0]).flatten()])


@pytest.mark.parametrize("paged", [False, True])
def test_prompted_rows_vs_oracle(moshi, paged):
    """Rows admitted with prompts at different ticks while others generate: P = 1 (< max_delay), P = 7, and P = 40 >
    context (the ring wraps inside the prefill).  The oracle is forced through the same prompt, then with our tokens; every
    decision after the prompt is the oracle's argmax within the margin rule."""
    m, w = moshi
    B, T = 4, 14
    plan = {0: (0, 7), 1: (2, 1), 2: (3, 40), 3: (1, 0)}           # row: (admission tick, P)
    seqs = {r: _seq(P + T, 40 + r) for r, (_, P) in plan.items()}
    x = torch.randint(0, CFG.card, (T, B, N_USER, 1), generator=torch.Generator().manual_seed(9))
    gen = LMGen(m, use_sampling=False)
    wb = {k: v.to(BF) for k, v in w.items()}
    ora, stats = {}, {r: [0, 0, 0.0] for r in plan}
    with gen.streaming(B, kv_pages=64 if paged else None), torch.no_grad():
        if paged:
            gen.reserve_kv(list(range(B)), 10 ** 6)          # whole rings: rows step before their admission too
        for t in range(T):
            new = [r for r, (a, _) in plan.items() if a == t]
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
            gen.step(x[t].to(DEV))
            CT = gen._st.cache.shape[2]
            for r, o in ora.items():
                ours = gen._st.cache[r:r + 1, :DQ + 1, int(gen._st.off_host[r]) % CT].cpu()
                o.step(x[t][r:r + 1], force=ours)
                d = _margin(o, ours)
                stats[r][0] += int((d == 0).sum()); stats[r][1] += d.numel(); stats[r][2] = max(stats[r][2], float(d.max()))
    for r, (exact, n, worst) in stats.items():
        print(f"row {r} (tick {plan[r][0]}, P = {plan[r][1]}): {exact}/{n} exact; worst deficit {worst:.3f}")
        assert n > 0 and worst <= 0.1 and exact >= 0.8 * n


def test_prefilled_row_continues_a_stepped_row(moshi):
    """Greedy LMGen stepped P frames from empty in row 0, recording what it sampled and was fed; row 1 prefilled with that
    prompt continues the run: its K/V within bf16 rounding of row 0's and its tokens those of row 0 under the margin rule."""
    m, w = moshi
    B, P, T = 2, 9, 8
    x = torch.randint(0, CFG.card, (P + T, 1, N_USER, 1), generator=torch.Generator().manual_seed(3))
    gen = LMGen(m, use_sampling=False)
    with gen.streaming(B), torch.no_grad():
        st = gen._st
        gen.set_active_streams([1, 0])
        prompt = torch.zeros(K, P, dtype=torch.int64)
        for t in range(P):
            gen.step(x[t].expand(B, -1, -1).to(DEV))
            prompt[:DQ + 1, t] = st.lm.tokens[0].cpu()
            prompt[DQ + 1:, t] = x[t][0, :, 0]
        gen.prefill_streams({1: prompt})
        assert list(st.off_host) == [P, P] and list(st.lm.pos_host) == [P, P]
        assert torch.equal(st.cache[0], st.cache[1]) and torch.equal(st.off, torch.full_like(st.off, P))
        for l in range(len(st.lm.kv)):
            a, b = st.lm.kv[l][:, 0, :, :P].float(), st.lm.kv[l][:, 1, :, :P].float()
            assert torch.allclose(a, b, rtol=2 ** -6, atol=2 ** -6), l
        gen.set_active_streams(None)
        same = n = 0
        for t in range(P, P + T):
            gen.step(x[t].expand(B, -1, -1).to(DEV))
            tk = st.lm.tokens.cpu()
            same += int((tk[0] == tk[1]).sum()); n += DQ + 1
            # later frames follow each row's own history: once they part, stop comparing
            if not torch.equal(tk[0], tk[1]):
                break
    print(f"{same}/{n} tokens of the prefilled row equal the stepped row's")
    assert same >= 0.8 * n


# ------------------------------------------------------------------------------------------- exact invariants
def _corpus(n, seed, Pmax=30, Gmax=12):
    g = np.random.default_rng(seed)
    out = []
    for i in range(n):
        P, G = int(g.integers(0, Pmax)), int(g.integers(1, Gmax))
        out.append((f"u{i}", _seq(P + G, 1000 * seed + i), P))
    return out


SAMP = Sampling(True, 0.7, 25, 0.0, 0.8, 250, 0.0)


def _gen_all(m, items, capacity, **kw):
    gen = LMGen(m, use_sampling=True)
    return dict(generate_many(gen, items, capacity, seeds={u: 17 + int(u[1:]) for u, _, _ in items}, **kw))


def test_generate_many_invariants(moshi):
    """Per-item outputs do not depend on admission order, the other items or the row (capacity fixed); paged equals
    contiguous bit for bit; shapes are [dep_q + 1, L - P]."""
    m, _ = moshi
    items = _corpus(9, 1)
    a = _gen_all(m, items, 4)
    assert set(a) == {u for u, _, _ in items}
    for u, seq, P in items:
        assert a[u].shape == (DQ + 1, seq.shape[1] - P) and a[u].dtype == torch.int64
    b = _gen_all(m, items[::-1], 4)
    c = _gen_all(m, items[3:5] + items[:3] + items[5:], 4, kv_pages=2, stats=(stats := {}))   # at most 2 live
    alone = {u: _gen_all(m, [it], 4)[u] for it in items[:3] for u in [it[0]]}
    for u in a:
        assert torch.equal(a[u], b[u]), u
        assert torch.equal(a[u], c[u]), u
    for u, v in alone.items():
        assert torch.equal(a[u], v), u
    assert stats["frames"] > 0 and stats["prefill_rows"] == sum(P for _, _, P in items)


def test_generate_many_p0_equals_hand_loop(moshi):
    m, _ = moshi
    items = [(f"u{i}", _seq(L, 70 + i), 0) for i, L in enumerate([6, 9, 4])]
    got = _gen_all(m, items, 3)
    gen = LMGen(m, use_sampling=True)
    with gen.streaming(3), torch.no_grad():
        gen.set_stream_sampling([])
        for r, (u, _, _) in enumerate(items):
            gen.reset_streaming(streams=[r])
            gen.set_stream_sampling([r], None, 17 + r)
        outs = {u: [] for u, _, _ in items}
        for t in range(9):
            act = [int(t < s.shape[1]) for _, s, _ in items]
            gen.set_active_streams(act)
            user = torch.stack([s[DQ + 1:, min(t, s.shape[1] - 1)] for _, s, _ in items])[:, :, None]
            gen.step(user.to(DEV))
            for r, (u, s, _) in enumerate(items):
                if act[r]:
                    outs[u].append(gen._st.out[r].cpu())
    for u, _, _ in items:
        assert torch.equal(got[u], torch.stack(outs[u], 1)), u


def test_prefill_leaves_other_rows_untouched(moshi):
    """A prompted admission changes no byte of the other rows' KV, counters or delay cache."""
    m, _ = moshi
    B = 3
    gen = LMGen(m, use_sampling=False)
    with gen.streaming(B), torch.no_grad():
        st = gen._st
        x = torch.randint(0, CFG.card, (B, N_USER, 1), generator=torch.Generator().manual_seed(1)).to(DEV)
        for _ in range(5):
            gen.step(x)
        snap = [t.clone() for t in st.lm.kv] + [st.cache.clone(), st.off.clone(), st.valid.clone(), st.lm.offset.clone(),
                                                 st.lm.row_step.clone()]
        gen.reset_streaming(streams=[1])
        gen.prefill_streams({1: prompt_from_aligned(_seq(30, 5), 30, CFG.delays, DQ)})
        after = [t for t in st.lm.kv] + [st.cache, st.off, st.valid, st.lm.offset, st.lm.row_step]
        for a, b in zip(snap, after):
            if a.dim() == 5:                      # kv [2, B, H, cap, hd]
                assert torch.equal(a[:, [0, 2]], b[:, [0, 2]])
            else:
                assert torch.equal(a[[0, 2]], b[[0, 2]])
        assert int(st.off[1]) == 30 and int(st.valid[1]) == 1 and int(st.lm.offset[1]) == 30 and st.off_host[1] == 30


# ------------------------------------------------------------------------------------------- serving
@pytest.fixture(scope="module")
def codec(official_weights):
    from rstnet_b200.codec import MimiCodec
    c = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    c.load_state_dict(official_weights, strict=True)
    c = c.to(DEV).eval()
    c.use_cuda_graphs, c.streaming_tensor_cores = True, True
    return c


def _audio(L, seed):
    return 0.1 * torch.randn(L, generator=torch.Generator().manual_seed(seed))


def _chunks(P, context=CFG.context):
    n, pos = 0, 0
    while pos < P:
        pos += row_chunk_positions(P - pos, 128, context, context, pos)
        n += 1
    return n


@pytest.mark.parametrize("paged", [False, True])
def test_scheduler_prompted_session(moshi, codec, paged):
    """A prompted session admitted next to a live one: held for exactly one tick per prefill chunk (its frames queue),
    then its first frames equal LMGen.prefill_streams + step in a bare scope of the same capacity and seed."""
    from rstnet_b200.serve import FrameScheduler, MoshiDuplexEngine
    m, _ = moshi
    B, P, ticks = 3, 20, 10
    prompt = prompt_from_aligned(_seq(P, 8), P, CFG.delays, DQ)
    eng = MoshiDuplexEngine(codec, LMGen(m, use_sampling=False), B, kv_pages=60 if paged else None)
    sch = FrameScheduler(eng, B)
    live = _audio(1920 * ticks, 1)
    mine = _audio(1920 * ticks, 2)
    sch.admit("live", seed=1)
    got, held = [], 0
    for t in range(ticks):
        if t == 1:
            r = sch.admit("p", seed=5, prompt=prompt)
        sch.push("live", live[1920 * t:1920 * (t + 1)])
        if t >= 1:
            sch.push("p", mine[1920 * (t - 1):1920 * t])
            held += r in eng.prefilling
        out = sch.tick()
        if t >= 1 and r not in eng.prefilling and "p" in out:
            got.append(out["p"])
        if t >= 1:
            assert ("p" in out) == (r not in eng.prefilling)
    n_chunks = _chunks(P)
    assert n_chunks > 1 and held == n_chunks        # the last chunk runs before its tick's step
    assert len(got) == ticks - n_chunks
    gen = LMGen(m, use_sampling=False)
    with codec.streaming(B), gen.streaming(B):
        gen.set_stream_sampling([r], None, 5)
        gen.prefill_streams({r: prompt})
        for i in range(len(got)):
            pcm = mine[1920 * i:1920 * (i + 1)].reshape(1, 1, -1).expand(B, 1, -1).contiguous().to(DEV)
            toks = gen.step(codec.encode(pcm))
            valid = gen.valid_rows()[r]
            if not valid:
                assert got[i] == (None, None)
                continue
            tk, p = got[i]
            assert torch.equal(tk, toks[r, :, 0].cpu()), i
            assert torch.equal(p, codec.decode(toks[:, 1:].clamp(0, 2047)).cpu()[r, 0]), i
    codec._stream_state = None


def test_scheduler_refuses_prompt_on_short_pool(moshi, codec):
    from rstnet_b200.serve import FrameScheduler, MoshiDuplexEngine
    m, _ = moshi
    eng = MoshiDuplexEngine(codec, LMGen(m, use_sampling=False), 2, kv_pages=3, kv_page=16)
    sch = FrameScheduler(eng, 2, kv_headroom=1)
    prompt = prompt_from_aligned(_seq(40, 1), 40, CFG.delays, DQ)           # 41 positions: pages_for -> 1 ring = 1 page
    with pytest.raises(RuntimeError, match="short"):
        FrameScheduler(eng, 2, kv_headroom=3).admit("p", prompt=prompt)
    assert eng.kv_pages_free == 3 and not eng.prefilling
    assert sch.admit("p", prompt=prompt) == 0
    codec._stream_state = None


def test_prompted_session_suspend_resume(moshi, codec):
    """A prompted session suspended and resumed in the engine gives the frames of an uninterrupted run."""
    from rstnet_b200.serve import FrameScheduler, MoshiDuplexEngine
    m, _ = moshi
    B, P, ticks = 2, 12, 8
    prompt = prompt_from_aligned(_seq(P, 3), P, CFG.delays, DQ)
    mine = _audio(1920 * ticks, 4)

    def run(suspend_at):
        eng = MoshiDuplexEngine(codec, LMGen(m, use_sampling=False), B, kv_pages=40)
        sch = FrameScheduler(eng, B)
        sch.admit("other", seed=2)
        sch.admit("p", seed=6, prompt=prompt)
        outs = []
        for t in range(ticks):
            sch.push("p", mine[1920 * t:1920 * (t + 1)])
            sch.push("other", mine[1920 * t:1920 * (t + 1)])
            if t == suspend_at:
                sch.suspend("p")
            if t == suspend_at + 2:
                sch.resume("p")
            outs += [v for s, v in sch.tick().items() if s == "p"]
        while sch._queue["p"]:
            outs += [v for s, v in sch.tick().items() if s == "p"]
        return outs
    a, b = run(-10), run(3)
    assert len(a) == len(b) == ticks
    for (ta, pa), (tb, pb) in zip(a, b):
        assert (ta is None) == (tb is None)
        if ta is not None:
            assert torch.equal(ta, tb) and torch.equal(pa, pb)
    codec._stream_state = None


# ------------------------------------------------------------------------------------------- CLI
def test_offline_continue(moshi, codec, official_weights, tmp_path):
    from rstnet_b200 import offline
    m, w = moshi
    cfg = tmp_path / "lm.json"
    cfg.write_text(json.dumps(CFG.reference_kwargs()))
    torch.save(w, tmp_path / "ckpt.pt")
    torch.save(official_weights, tmp_path / "codec.pt")
    corpus = {f"d{i}": _seq(L, 300 + i) for i, L in enumerate([20, 30, 25])}
    torch.save(corpus, tmp_path / "corpus.pt")
    P = 8
    rc = offline.main(["continue", "--model", "moshi", "--config", str(cfg), "--checkpoint", str(tmp_path / "ckpt.pt"),
                       "--input", str(tmp_path / "corpus.pt"), "--prompt-frames", str(P), "--output-file",
                       str(tmp_path / "out.pt"), "--capacity", "2", "--seed", "3", "--wav-dir", str(tmp_path / "wav"),
                       "--codec-checkpoint", str(tmp_path / "codec.pt")])
    assert rc == 0
    out = torch.load(tmp_path / "out.pt")
    gen = LMGen(m, use_sampling=True, temp=0.8, temp_text=0.7, top_k=250, top_k_text=25)
    want = dict(generate_many(gen, [(u, s, P) for u, s in corpus.items()], 2, seeds={u: 3 for u in corpus}))
    assert set(out) == set(want)
    for u in want:
        assert torch.equal(out[u], want[u]), u
    j0 = max(0, MD - P)
    import argparse
    codec = offline._load_codec(argparse.Namespace(weights=str(tmp_path / "codec.pt"), config=None, device=DEV))
    wavs = dict(codec.decode_many([(u, o[1:DQ + 1, j0:].clamp(0, 2047)) for u, o in want.items()], 64))
    for u, wv in wavs.items():
        got, sr = offline.read_wav(str(tmp_path / "wav" / f"{u}_sample.wav"))
        assert sr == 24000 and got.shape == wv.shape
        assert float((got - wv.clamp(-1, 1)).abs().max()) <= 2.0 / 32767
