"""Paged KV cache (-m gpu): the paged entry points of the RoPE/KV-append and ring decode attention kernels against their
contiguous forms on the same data, a paged GPT.streaming scope against a contiguous one, and InferenceImp.generate_many
on a pool shorter than its capacity against InferenceImp.generate on each utterance alone.  Paging changes addresses
only, so every comparison is bit for bit."""
import random

import numpy as np
import pytest
import torch

from oracle import lm_oracle as L
from rstnet_b200 import _lib, ops
from rstnet_b200._lib import RstnetError
from rstnet_b200.lm import GPT, Config

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
BF = torch.bfloat16
TEXT_EMPTY = 128002
SENTINEL = 1234.0   # every pool row no stream maps (a kernel that wrote there would change it)
bits = lambda t: t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------------ 1. kernels
def _paged_copy(kv, table, page, n_pages):
    """The pool [n_pages, 2, n_kv, page, hs] holding the contiguous rings kv [2, B, n_kv, cap, hs] at the pages of `table`
    [B, stride]; every other row holds SENTINEL."""
    _, B, nkv, cap, hs = kv.shape
    pool = torch.full((n_pages, 2, nkv, page, hs), SENTINEL, dtype=BF, device=DEV)
    for b in range(B):
        for i, p in enumerate(table[b].tolist()):
            n = min(page, cap - i * page)
            if p >= 0 and n > 0:
                pool[p, :, :, :n] = kv[:, b, :, i * page:i * page + n]
    return pool


def _gather(pool, table, cap):
    """The contiguous rings [2, B, n_kv, cap, hs] read back through the table (unmapped pages as NaN)."""
    n_pages, _, nkv, page, hs = pool.shape
    B = table.shape[0]
    out = torch.full((2, B, nkv, cap, hs), float("nan"), dtype=BF, device=DEV)
    for b in range(B):
        for i, p in enumerate(table[b].tolist()):
            n = min(page, cap - i * page)
            if p >= 0 and n > 0:
                out[:, b, :, i * page:i * page + n] = pool[p, :, :, :n]
    return out


def _untouched_mask(table, page, cap, n_pages):
    """Pool rows no stream maps: unassigned pages and the rows of a last page past the ring."""
    keep = torch.ones(n_pages, page, dtype=torch.bool)
    for b in range(table.shape[0]):
        for i, p in enumerate(table[b].tolist()):
            if p >= 0:
                keep[p, :max(0, min(page, cap - i * page))] = False
    return keep


def _launch(paged, qkv, cos, sin, offset, rs, rt, q, kv, att, M, B, nh, nkv, hs, cap, context, pt=None, stride=0, log2=0):
    lib, st = _lib.lib(), ops._stream()
    rp = (rs.data_ptr(), rt.data_ptr()) if rs is not None else (None, None)
    head = (qkv.data_ptr(), cos.data_ptr(), sin.data_ptr(), cos.shape[0], cos.shape[1], offset.data_ptr(), 1, *rp, q.data_ptr(),
            kv.data_ptr(), M, B, nh, nkv, hs, cap)
    ahead = (q.data_ptr(), kv.data_ptr(), offset.data_ptr(), 1, *rp, att.data_ptr(), M, B, nh, nkv, hs, cap, context)
    if paged:
        _lib.check(lib.rstnet_lm_rope_kv_append_paged_bf16(*head, pt.data_ptr(), stride, log2, st))
        _lib.check(lib.rstnet_lm_paged_decode_attention_bf16(*ahead, pt.data_ptr(), stride, log2, st))
    else:
        _lib.check(lib.rstnet_lm_rope_kv_append_bf16(*head, st))
        _lib.check(lib.rstnet_lm_ring_decode_attention_bf16(*ahead, st))


@pytest.mark.parametrize("nh,nkv,hs,rope_n", [(4, 4, 64, 64), (4, 4, 128, 128), (8, 2, 128, 96), (6, 2, 64, 32)])
@pytest.mark.parametrize("form", ["decode", "multi", "rows"])
def test_paged_kernels_equal_contiguous(nh, nkv, hs, rope_n, form):
    """Pages of 16 over a ring of 56 (its last page half used), assigned scrambled and interleaved across streams; streams
    before and after their ring wraps."""
    g = torch.Generator().manual_seed(nh * 1000 + hs + rope_n)
    B, cap, page, log2, n_pages, rope_rows = 5, 56, 16, 4, 29, 128
    stride = -(-cap // page)
    context = cap
    qpk = nh // nkv
    tn = 1 if form == "decode" else 3
    offset = torch.tensor([2, 70, 30, 53, 0] if tn > 1 else [2, 70, 55, 56, 111], dtype=torch.int64, device=DEV)
    table = torch.randperm(n_pages, generator=g)[:B * stride].view(stride, B).t().contiguous().to(torch.int32)
    pt = table.to(DEV)
    kv0 = torch.randn(2, B, nkv, cap, hs, generator=g).to(DEV, BF)
    cos = torch.randn(rope_rows, rope_n, generator=g).to(DEV, BF)
    sin = torch.randn(rope_rows, rope_n, generator=g).to(DEV, BF)
    if form == "rows":
        pairs = [(b, t) for b in (0, 1, 3) for t in range(tn)]
        random.Random(hs).shuffle(pairs)
        rows = pairs[:4] + [(-1, 0)] * 2 + pairs[4:] + [(-1, 0)]
        rs = torch.tensor([b for b, _ in rows], dtype=torch.int32, device=DEV)
        rt = torch.tensor([t for _, t in rows], dtype=torch.int32, device=DEV)
    else:
        rows = [(r % B, r // B) for r in range(tn * B)]
        rs = rt = None
    M = len(rows)
    qkv = torch.randn(M, nkv * (qpk + 2) * hs, generator=g).to(DEV, BF)
    nan = float("nan")
    kv_c, pool = kv0.clone(), _paged_copy(kv0, table, page, n_pages)
    keep = _untouched_mask(table, page, cap, n_pages)
    outs = {}
    for paged, kv in ((False, kv_c), (True, pool)):
        q = torch.full((M, nh * hs), nan, dtype=BF, device=DEV)
        att = torch.full((M, nh * hs), nan, dtype=BF, device=DEV)
        _launch(paged, qkv, cos, sin, offset, rs, rt, q, kv, att, M, B, nh, nkv, hs, cap, context, pt, stride, log2)
        outs[paged] = (q, att)
    torch.cuda.synchronize()
    assert torch.equal(bits(outs[True][0]), bits(outs[False][0]))
    assert torch.equal(bits(outs[True][1]), bits(outs[False][1]))
    assert all(torch.isnan(outs[True][1][r].float()).all() for r, (b, _) in enumerate(rows) if b < 0)   # padding rows
    assert torch.equal(bits(_gather(pool, table, cap)), bits(kv_c))
    assert bool((pool.permute(0, 3, 1, 2, 4)[keep.to(DEV)] == SENTINEL).all())


def test_unmapped_rows_write_nothing_and_output_zeros():
    """A stream whose own position falls on an unmapped page (a held stream without pages, or one past its pages) writes
    no K/V and no q, and its attention output is zeros; the other streams are unaffected."""
    g = torch.Generator().manual_seed(5)
    B, nh, nkv, hs, cap, page, log2, n_pages = 4, 8, 2, 128, 48, 16, 4, 12
    stride = 3
    table = torch.arange(B * stride, dtype=torch.int32).view(B, stride)
    table[1] = -1                 # no pages at all
    table[2, 1:] = -1             # only slots 0..15; its position 20 is on an unmapped page
    offset = torch.tensor([5, 0, 20, 40], dtype=torch.int64, device=DEV)
    kv0 = torch.randn(2, B, nkv, cap, hs, generator=g).to(DEV, BF)
    cos = torch.randn(64, hs, generator=g).to(DEV, BF)
    sin = torch.randn(64, hs, generator=g).to(DEV, BF)
    qkv = torch.randn(B, nkv * (nh // nkv + 2) * hs, generator=g).to(DEV, BF)
    pool = _paged_copy(kv0, table, page, n_pages)
    before = pool.clone()
    kv_c = kv0.clone()
    outs = {}
    for paged, kv in ((False, kv_c), (True, pool)):
        q = torch.full((B, nh * hs), float("nan"), dtype=BF, device=DEV)
        att = torch.full((B, nh * hs), float("nan"), dtype=BF, device=DEV)
        _launch(paged, qkv, cos, sin, offset, None, None, q, kv, att, B, B, nh, nkv, hs, cap, cap, table.to(DEV), stride, log2)
        outs[paged] = (q, att)
    torch.cuda.synchronize()
    q, att = outs[True]
    for b in (1, 2):
        assert torch.isnan(q[b].float()).all(), b
        assert bool((att[b].float() == 0).all()) and not torch.signbit(att[b].float()).any(), b
    for b in (0, 3):
        assert torch.equal(bits(q[b]), bits(outs[False][0][b])) and torch.equal(bits(att[b]), bits(outs[False][1][b])), b
    changed = (bits(pool) != bits(before)).any(dim=-1)          # [n_pages, 2, n_kv, page]
    written = {(int(p), int(r)) for p, _, _, r in changed.nonzero().tolist()} if changed.any() else set()
    expect = {(int(table[b, (int(offset[b]) % cap) // page]), (int(offset[b]) % cap) % page) for b in (0, 3)}
    assert written <= expect


def test_bad_page_arguments_fail_before_launch():
    lib, st = _lib.lib(), ops._stream()
    B, nh, nkv, hs, cap = 2, 4, 4, 64, 40
    z = lambda *s, dt=BF: torch.zeros(*s, dtype=dt, device=DEV)
    qkv, q, att = z(B, nkv * 3 * hs), z(B, nh * hs), z(B, nh * hs)
    cos = sin = z(64, hs)
    offset = z(B, dt=torch.int64)
    pool = z(8, 2, nkv, 16, hs)
    pt = torch.zeros(B, 4, dtype=torch.int32, device=DEV)
    n0 = _lib.launch_count()
    for ptr, stride, log2 in ((pt.data_ptr(), 4, 3), (pt.data_ptr(), 4, 13), (pt.data_ptr(), 2, 4), (None, 3, 4),
                              (pt.data_ptr(), 0, 4)):
        assert lib.rstnet_lm_rope_kv_append_paged_bf16(qkv.data_ptr(), cos.data_ptr(), sin.data_ptr(), 64, hs, offset.data_ptr(), 1,
                                                       None, None, q.data_ptr(), pool.data_ptr(), B, B, nh, nkv, hs, cap, ptr,
                                                       stride, log2, st) != 0
        assert lib.rstnet_lm_paged_decode_attention_bf16(q.data_ptr(), pool.data_ptr(), offset.data_ptr(), 1, None, None,
                                                         att.data_ptr(), B, B, nh, nkv, hs, cap, cap, ptr, stride, log2, st) != 0
    assert _lib.launch_count() == n0


# ------------------------------------------------------------------------------------------------------ 2. scope
def _gpt(context, block_size=64):
    cfg = L.SMALL
    w32 = L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05)
    m = GPT(Config(block_size=block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                   intermediate_size=cfg.intermediate_size, norm_eps=cfg.norm_eps, padded_vocab_size=cfg.padded_vocab_size,
                   audio_card=cfg.audio_card, n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim,
                   codecformer_heads=cfg.codecformer_heads, codecformer_layers=cfg.codecformer_layers,
                   codecformer_dim_feedforward=cfg.codecformer_dim_feedforward, context=context))
    m.load_state_dict(w32, strict=True)
    return m.to(DEV, BF).eval()


@pytest.fixture(scope="module")
def lm40():
    """context 40 (rings wrap within the 64 positions of block_size), pages of 16: three per ring, the last half used."""
    return _gpt(40)


def _ids(g, *shape):
    x = torch.randint(0, 2048, shape, generator=g)
    x[..., 0, :] = torch.randint(0, 1000, x[..., 0, :].shape, generator=g)
    return x.to(DEV)


def test_paged_scope_equals_contiguous_scope(lm40):
    """The same calls on a contiguous scope and on a paged one (pool of 12 pages of 16): a prefill, forward_step frames
    past the ring's wrap, held rows without pages, prefill_streams admissions mid-run and a parked and resumed scope.  The
    active rows' tokens, transformer_out and text logits match bit for bit."""
    m = lm40
    B = 4
    g = torch.Generator().manual_seed(3)
    script = []    # (op, args) replayed on both scopes
    script.append(("reserve", ([0, 1, 2], 64)))
    script.append(("reserve", ([3], 30)))
    script.append(("prefill", _ids(g, B, 9, 5)))
    script += [("step", _ids(g, B, 9, 1)) for _ in range(12)]
    script.append(("active", [1, 1, 1, 0]))
    script.append(("release", [3]))
    script += [("step", _ids(g, B, 9, 1)) for _ in range(4)]
    script.append(("reset", [3]))
    script.append(("reserve", ([3], 36)))
    script.append(("prompts", {3: _ids(g, 9, 7), 1: _ids(g, 9, 3)}))
    script.append(("active", [1, 1, 1, 1]))
    script += [("step", _ids(g, B, 9, 1)) for _ in range(8)]
    script.append(("park", None))
    script += [("step", _ids(g, B, 9, 1)) for _ in range(8)]
    script.append(("active", [1, 1, 0, 1]))
    script += [("step", _ids(g, B, 9, 1)) for _ in range(8)]

    def run(kv_pages):
        got = []
        active = np.ones(B, dtype=bool)
        with m.streaming(B, kv_pages=kv_pages, kv_page=16):
            for op, a in script:
                if op in ("reserve", "release") and kv_pages is None:
                    continue
                if op == "reserve":
                    m.reserve_kv(*a)
                elif op == "release":
                    m.release_kv(a)
                elif op == "prefill":
                    out, logits = m.forward_global(a)
                    got.append((out.clone(), logits.clone(), active.copy()))
                elif op == "step":
                    toks = m.forward_step(a)
                    st = m._state
                    got.append((toks.clone(), st.out.clone(), st.logits.clone(), active.copy()))
                elif op == "active":
                    active = np.array(a, dtype=bool)
                    m.set_active_streams(a)
                elif op == "reset":
                    m.reset_streaming(streams=a)
                elif op == "prompts":
                    m.prefill_streams(a)
                elif op == "park":
                    saved = m.get_streaming_state()
                    with m.streaming(2):    # another scope runs in between
                        m.forward_step(_ids(torch.Generator().manual_seed(9), 2, 9, 1))
                    m.set_streaming_state(saved)
            m.check_device_errors()
            if kv_pages is not None:
                assert m.kv_pages_free == kv_pages - 4 * 3
        return got

    ref, pag = run(None), run(12)
    assert len(ref) == len(pag) > 40
    for i, (r, p) in enumerate(zip(ref, pag)):
        act = torch.from_numpy(r[-1]).to(DEV)
        assert np.array_equal(r[-1], p[-1])
        for a, b in zip(r[:-1], p[:-1]):
            a, b = a.view(B, -1), b.view(B, -1)
            assert torch.equal(bits(a[act]) if a.dtype == BF else a[act], bits(b[act]) if b.dtype == BF else b[act]), i


def test_reservation_guard_raises_before_launch(lm40):
    m = lm40
    B = 3
    g = torch.Generator().manual_seed(4)
    with m.streaming(B, kv_pages=6, kv_page=16):
        assert m.kv_page_bytes == m.config.n_layer * 2 * m.config.n_query_groups * 16 * m.config.head_size * 2
        m.reserve_kv([0, 1], [64, 6])          # stream 2: no pages
        m.set_active_streams([1, 1, 0])        # a held stream needs none
        m.prefill(_ids(g, B, 9, 4))
        for _ in range(2):
            m.forward_step(_ids(g, B, 9, 1))
        st = m._state
        off, pos = st.offset.clone(), st.pos_host.copy()
        n0 = _lib.launch_count()
        with pytest.raises(RstnetError):
            m.forward_step(_ids(g, B, 9, 1))    # stream 1 would write position 6 of 6
        with pytest.raises(RstnetError):
            m.prefill(_ids(g, B, 9, 2))
        with pytest.raises(RstnetError):
            m.prefill_streams({1: _ids(g, 9, 1)})
        m.set_active_streams([1, 0, 1])
        with pytest.raises(RstnetError):
            m.forward_step(_ids(g, B, 9, 1))    # stream 2 holds no pages
        torch.cuda.synchronize()
        assert _lib.launch_count() == n0
        assert torch.equal(st.offset, off) and np.array_equal(st.pos_host, pos)
        with pytest.raises(RstnetError):
            m.reserve_kv([2], 64 * 16)          # 3 more pages, 2 free: nothing changes
        assert m.kv_pages_free == 2 and np.array_equal(st.pages.table[2], [-1, -1, -1])
        m.reserve_kv([1], 40)                   # grows in place: the written positions keep their pages
        m.set_active_streams([1, 1, 0])
        m.forward_step(_ids(g, B, 9, 1))
        m.check_device_errors()
    with m.streaming(B):
        for call in (lambda: m.reserve_kv([0], 4), lambda: m.release_kv([0]), lambda: m.kv_pages_free,
                     lambda: m.kv_page_bytes):
            with pytest.raises(RstnetError):
                call()


# ------------------------------------------------------------------------------------------------------ 3. generate_many
def _corpus(n, seed, pmax, gmax):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        P = int(torch.randint(3, pmax + 1, (1,), generator=g))
        G = int(torch.randint(2, gmax + 1, (1,), generator=g))
        seq = torch.randint(0, 2048, (9, P + G), generator=g)
        seq[0, :P] = torch.randint(0, 1000, (P,), generator=g)
        seq[0, P:] = TEXT_EMPTY
        out.append((f"utt{i}", seq))
    return out


def _imp(m):
    from rstnet_b200.infer import InferenceImp
    return InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")


def test_generate_many_short_pool_equals_each_utterance_alone():
    """context 200 (4 pages of 64 per ring) and utterances of 5..140 positions (1..3 pages): a pool of 6 pages holds 2-3
    of them at once, at capacities 4 and 7."""
    m = _gpt(200, block_size=256)
    imp = _imp(m)
    corpus = _corpus(14, 11, 40, 100)
    alone = {}
    for utt, seq in corpus:
        codes, raw = imp.generate(seq.unsqueeze(0).to(DEV), return_frames=True)
        alone[utt] = (codes[0].cpu(), raw[0].cpu())
    orders = []
    for cap, pool in ((4, 6), (7, 6), (7, 6), (4, None)):
        stats = {}
        got = list(imp.generate_many(((u, s.to(DEV)) for u, s in corpus), cap, return_frames=True, kv_pages=pool, stats=stats))
        assert sorted(u for u, _, _ in got) == sorted(u for u, _ in corpus)
        for utt, codes, raw in got:
            assert torch.equal(codes.cpu(), alone[utt][0]), (cap, utt)
            assert torch.equal(raw.cpu(), alone[utt][1]), (cap, utt)
        if pool is not None:
            assert stats["wait_frames"] > 0
        orders.append([u for u, _, _ in got])
    assert orders[1] == orders[2]           # the same pool: the same completion order
    big = torch.randint(0, 2048, (9, 200), generator=torch.Generator().manual_seed(12))   # P 30 + G 170: 4 pages
    big[0, :30] = torch.randint(0, 1000, (30,), generator=torch.Generator().manual_seed(13))
    big[0, 30:] = TEXT_EMPTY
    with pytest.raises(RstnetError):
        list(imp.generate_many([("big", big.to(DEV))], 2, kv_pages=3))


def test_generate_many_capacity_130_short_pool():
    """The 256-column GEMM's width (130 rows) on a pool of 100 one-page rings (context 16): utterances wait for pages."""
    m = _gpt(16)
    imp = _imp(m)
    corpus = _corpus(150, 13, 10, 6)
    stats = {}
    got = {u: (c, r) for u, c, r in imp.generate_many(((u, s.to(DEV)) for u, s in corpus), 130, return_frames=True,
                                                      kv_pages=100, stats=stats)}
    assert sorted(got) == sorted(u for u, _ in corpus) and stats["wait_frames"] > 0
    for utt, seq in corpus[::7]:
        codes, raw = imp.generate(seq.unsqueeze(0).to(DEV), return_frames=True)
        assert torch.equal(got[utt][0].cpu(), codes[0].cpu()), utt
        assert torch.equal(got[utt][1].cpu(), raw[0].cpu()), utt
