"""LM decode attention (-m gpu) in every launch form the models use, against a float64 softmax over exactly the positions
each query may attend: multi-position prefill chunks at the lengths lm.prefill_chunk and lm.row_chunk_positions choose,
ragged row maps with padding rows, paged pools, and the Moshi scoring scope's 3000-position window.

A row at position p attends positions max(0, p - context + 1, p + 2 - cap) .. p, the single-step decode window
(test_lm_kernels_gpu.ring_keys), which every chunk must equal.  The reference keeps one K/V per position and reads the
window by position; the ring is built by replaying the appends (slot s of a stream holds its latest position of the
launch with position % cap == s).  So a query whose window slot was overwritten by a later position of the same launch
reads another value than the reference: that is the overwrite the chunk lengths must prevent.

Three traps make a wrong key visible even where one key among 3000 barely moves a mean:

* every ring slot whose position no row of the launch attends is NaN in K and V (empty slots, stale positions, the
  ring-quirk slot p + 1 - cap and position p - context included): reading one turns that row's output into NaN;
* every position of a chunk after its first is a key K = 8u, V = 1000, with the queries of a KV group all along u: a
  later key of the same chunk leaking into an earlier row lands far outside the bound;
* pages no stream maps hold 1234, and output bytes no row owns (padding rows, past the last row) hold a NaN sentinel
  that must survive bit for bit.

Every output is held to test_lm_kernels_gpu's per-element bound |out - ref64| <= ulp_bf16(ref64) + 2^-12 * max |v| over
the attended keys, and to its bit-equal floor.  The bound needs no extra slack at 3000 keys: fp32 online-softmax sums
over n keys drift by about n * 2^-24 relative in the worst case, 1.8e-4 at n = 3000, inside 2^-12.
"""
import math

import pytest
import torch

import test_lm_kernels_gpu as KT
from rstnet_b200 import _lib, ops
from rstnet_b200.lm import KV_PAGE, MAX_ROWS, ROW_BUCKETS, prefill_chunk, row_chunk_positions

pytestmark = pytest.mark.gpu
DEV, BF, F64 = "cuda", torch.bfloat16, torch.float64
NAN = float("nan")
SENT = 0x7FA5          # bf16 NaN with a payload the kernel never writes: output bytes no row owns
UNMAPPED = 1234.0      # pool rows no stream maps
CHUNK_V = 1000.0       # V of the keys a chunk appends after its first position
TAIL = 2               # output rows past the last row
MOSHI_CONTEXT = 3000
MOSHI_CAP = MOSHI_CONTEXT + MAX_ROWS - 1     # moshi.LMModel._scratch_state's rings
LAYOUTS = {   # q_per_kv -> (n_head, n_kv) at hs 64 and 128
    1: (8, 8), 2: (8, 4), 3: (12, 4), 4: (16, 4), 8: (16, 2)}


# ------------------------------------------------------------------------------------------------------- launch shapes
def window_lo(p: int, cap: int, context: int) -> int:
    return max(0, p - context + 1, p + 2 - cap)


def uniform_chunk(pos, left, cap, context):
    """GPT.forward_global's prefill chunk for streams at positions `pos`: tn = lm.prefill_chunk, rows time-major
    (row tl * B + b)."""
    B = len(pos)
    tn = prefill_chunk(max(1, MAX_ROWS // B), left, cap, context, max(pos))
    assert tn > 1, "a multi-position chunk"
    return dict(B=B, start=list(pos), rows=[(r % B, r // B) for r in range(tn * B)], mapped=False, cap=cap, context=context)


def ragged_chunk(pos, left, cap, context, pad_after=(), reverse=(), idle=0):
    """_LMState.row_chunk's packing of streams at positions `pos` with `left` positions to feed: each stream's length
    from lm.row_chunk_positions within the MAX_ROWS budget, in order.  Padding rows (-1) follow the streams listed in
    `pad_after` and fill the launch up to the next row bucket (at least one); streams in `reverse` list their rows last
    position first; `idle` more streams have rings but no rows."""
    rows = []
    used = 0
    for s, (p, n) in enumerate(zip(pos, left)):
        budget = MAX_ROWS - used
        if budget == 0:
            break
        tn = row_chunk_positions(n, budget, cap, context, p)
        tls = range(tn - 1, -1, -1) if s in reverse else range(tn)
        rows += [(s, t) for t in tls]
        used += tn
        if s in pad_after:
            rows += [(-1, 0)] * 2
    end = next((b for b in ROW_BUCKETS if b > len(rows)), len(rows) + 1)
    rows += [(-1, 0)] * (end - len(rows))
    return dict(B=len(pos) + idle, start=list(pos) + [5 * cap + 7] * idle, rows=rows, mapped=True, cap=cap, context=context)


CASES = {
    # GPT prefill chunks (uniform rows): one empty stream up to MAX_ROWS positions; one long-wrapped stream at exactly
    # cap - context + 1 positions; 8 streams at every fill level (empty, partly filled, wrapping inside the chunk, just
    # wrapped, long wrapped) after the wrap; 8 streams with a full-ring window (context == cap) whose chunk ends exactly at
    # the wrap; 64 streams x 2 positions.  cap 72 is no multiple of a page.
    "b1_empty": lambda: uniform_chunk([0], 300, 200, 200),
    "b1_wrapped": lambda: uniform_chunk([1000], 300, 160, 40),
    "b8_mixed": lambda: uniform_chunk([0, 5, 37, 60, 63, 72, 300, 1000], 40, 72, 64),
    "b8_to_wrap": lambda: uniform_chunk([56, 0, 10, 20, 30, 33, 40, 55], 40, 72, 72),
    "b64_tn2": lambda: uniform_chunk([(37 * b * b + 11 * b) % 600 for b in range(64)], 40, 48, 47),
    # ragged chunks (row maps): streams before, across and long after the wrap with context < cap (cap - context + 1
    # positions after the wrap) and with context == cap (a stream runs up to the wrap, cap - pos positions)
    "ragged": lambda: ragged_chunk([0, 30, 95, 99, 400, 2000], [20, 5, 40, 3, 30, 12], 100, 92, pad_after=(0, 3), reverse=(1,)),
    "ragged_full": lambda: ragged_chunk([0, 30, 95, 99, 400, 2000], [20, 5, 40, 3, 30, 12], 100, 100, pad_after=(2,), reverse=(0,)),
    # Moshi's scoring scope: 128-row chunks of one stream before the wrap, across it and far past it (every row then
    # attends 3000 keys), and of mixed streams around position 10000 with an idle stream
    "moshi_start": lambda: uniform_chunk([0], 10 ** 4, MOSHI_CAP, MOSHI_CONTEXT),
    "moshi_wrap": lambda: uniform_chunk([3050], 10 ** 4, MOSHI_CAP, MOSHI_CONTEXT),
    "moshi_10000": lambda: uniform_chunk([10000], 10 ** 4, MOSHI_CAP, MOSHI_CONTEXT),
    "moshi_mixed": lambda: ragged_chunk([9990, 10007, 12345, 3127], [50, 30, 100, 100], MOSHI_CAP, MOSHI_CONTEXT, pad_after=(1,),
                                        idle=1),
}


# ------------------------------------------------------------------------------------------------------------- driver
def _pool(ring, log2_page, g):
    """The rings [2, B, n_kv, cap, hs] in a pool of pages of 2^log2_page positions, assigned in a scrambled order
    interleaved across streams; one page whose slots no row reads is left unmapped.  -> (pool, table, pages_stride)"""
    _, B, nkv, cap, hs = ring.shape
    P = 1 << log2_page
    stride = -(-cap // P)
    n_pages = B * stride + 2
    table = torch.randperm(n_pages, generator=g)[:B * stride].view(stride, B).t().contiguous().to(torch.int32)
    dead = ring[0, :, 0, :, 0].isnan().cpu()          # [B, cap]: slots no row reads
    hole = next(((b, i) for b in range(B) for i in range(stride) if bool(dead[b, i * P:(i + 1) * P].all())), None)
    assert hole is not None, "no page outside every window to leave unmapped"
    table[hole] = -1
    pool = torch.full((n_pages, 2, nkv, P, hs), UNMAPPED, dtype=BF, device=DEV)
    for b in range(B):
        for i, p in enumerate(table[b].tolist()):
            n = min(P, cap - i * P)
            if p >= 0:
                pool[p, :, :, :n] = ring[:, b, :, i * P:i * P + n]
    return pool, table.to(DEV), stride


def run_case(name, case, nh, nkv, hs, dist, seed, log2_page=None, ostride=1):
    B, start, rows, cap, context = case["B"], case["start"], case["rows"], case["cap"], case["context"]
    M, rep = len(rows), nh // nkv
    g = torch.Generator(device=DEV).manual_seed(seed)
    u = torch.randn(nkv, hs, generator=g, device=DEV, dtype=F64)
    u = u / u.norm(dim=-1, keepdim=True)               # one query direction per KV group
    # K/V per position, the ring by replaying the appends, NaN in every slot no row attends
    ring = torch.full((2, B, nkv, cap, hs), NAN, dtype=BF, device=DEV)
    streams = []
    for b in range(B):
        idx = [r for r, (s, _) in enumerate(rows) if s == b]
        tls = torch.tensor([rows[r][1] for r in idx], dtype=torch.int64)
        last = start[b] + int(tls.max()) if idx else start[b] - 1      # the stream's last position in the launch
        kept = max(0, last - cap + 1)                                     # the oldest position its ring still holds
        wlo = window_lo(start[b], cap, context) if idx else last + 1     # the oldest position a row of it attends
        base = min(wlo, kept)
        kp = torch.randn(nkv, last - base + 1, hs, generator=g, device=DEV).to(BF)
        vp = torch.randn(nkv, last - base + 1, hs, generator=g, device=DEV).to(BF)
        if idx:
            kp[:, start[b] + 1 - base:] = (8 * u).to(BF)[:, None]
            vp[:, start[b] + 1 - base:] = CHUNK_V
        lo = max(wlo, kept)
        slots = torch.arange(lo, last + 1, device=DEV) % cap
        ring[0, b][:, slots], ring[1, b][:, slots] = kp[:, lo - base:], vp[:, lo - base:]
        streams.append((idx, tls, base, kp, vp))
    coef = {"random": lambda: 0.5 + torch.rand(M, nh, generator=g, device=DEV, dtype=F64),     # scores ~ N(0, 1)
            "sharp": lambda: 10 * (0.8 + 0.4 * torch.rand(M, nh, generator=g, device=DEV, dtype=F64)),   # about +-30
            "flat": lambda: torch.zeros(M, nh, device=DEV, dtype=F64)}[dist]() * math.sqrt(hs)
    q = (coef[:, :, None] * u.repeat_interleave(rep, 0)[None]).to(BF)    # head h = group h // rep
    pad = torch.tensor([s < 0 for s, _ in rows], device=DEV)
    q[pad] = NAN

    # float64 reference over each row's window, read by position
    ref = torch.full((M, nh, hs), NAN, dtype=F64, device=DEV)
    slack = torch.zeros(M, nh, 1, dtype=F64, device=DEV)
    for b, (idx, tls, base, kp, vp) in enumerate(streams):
        if not idx:
            continue
        p = start[b] + tls.to(DEV)
        lo = torch.clamp(torch.maximum(p - context + 1, p + 2 - cap), min=0)
        P = base + torch.arange(kp.shape[1], device=DEV)
        mask = (P[None] >= lo[:, None]) & (P[None] <= p[:, None])                       # [rows, positions]
        for t in (0, len(idx) - 1):      # the window is the single-step decode window
            assert sorted((P[mask[t]] % cap).tolist()) == sorted(KT.ring_keys(int(p[t]), cap, context).tolist())
        s = torch.einsum("tgjd,gnd->tgjn", q[idx].to(F64).view(-1, nkv, rep, hs), kp.to(F64)) * hs ** -0.5
        s = s.masked_fill(~mask[:, None, None], -math.inf)
        ref[idx] = torch.einsum("tgjn,gnd->tgjd", torch.softmax(s, -1), vp.to(F64)).reshape(-1, nh, hs)
        vmax = torch.where(mask[:, None], vp.to(F64).abs().amax(-1)[None], 0.0).amax(-1)     # [rows, n_kv]
        slack[idx] = KT.ATTN_C * vmax.repeat_interleave(rep, 1)[..., None]

    lib, st = _lib.lib(), ops._stream()
    off = torch.tensor(start if ostride else start[:1], dtype=torch.int64, device=DEV)
    if case["mapped"]:
        rs = torch.tensor([s for s, _ in rows], dtype=torch.int32, device=DEV)
        rt = torch.tensor([t for _, t in rows], dtype=torch.int32, device=DEV)
        rp = (rs.data_ptr(), rt.data_ptr())
    else:
        rp = (None, None)

    def launch(kv, pages=()):
        out = torch.full(((M + TAIL) * nh * hs,), SENT, dtype=torch.int16, device=DEV)
        args = (q.data_ptr(), kv.data_ptr(), off.data_ptr(), ostride, *rp, out.data_ptr(), M, B, nh, nkv, hs, cap, context)
        if pages:
            _lib.check(lib.rstnet_lm_paged_decode_attention_bf16(*args, *pages, st))
        else:
            _lib.check(lib.rstnet_lm_ring_decode_attention_bf16(*args, st))
        return out.view(M + TAIL, nh * hs)

    def check(label, out):
        torch.cuda.synchronize()
        real = ~pad
        KT.check_bound(f"{label} {name} nh {nh} n_kv {nkv} hs {hs} {dist} rows {M}", out[:M][real].view(BF).view(-1, nh, hs),
                       ref[real], slack[real], 0.98)
        owned = torch.cat([real, torch.zeros(TAIL, dtype=torch.bool, device=DEV)])
        assert bool((out[~owned] == SENT).all()), "output bytes of padding rows or past the last row were written"

    out = launch(ring)
    check("ring attention", out)
    if log2_page is not None:
        pool, table, stride = _pool(ring, log2_page, torch.Generator().manual_seed(seed))
        out_p = launch(pool, (table.data_ptr(), stride, log2_page))
        check(f"paged attention (page {1 << log2_page})", out_p)
        assert torch.equal(out_p, out), "the paged form must equal the contiguous ring bit for bit"


# -------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("hs", [64, 128])
@pytest.mark.parametrize("q_per_kv", [1, 2, 3, 4, 8])
def test_head_layouts_prefill_chunk(q_per_kv, hs):
    """Every head layout (G = 2 instantiations for even q_per_kv, G = 1 for odd, MHA and 8 heads per KV group) on the
    8-stream prefill chunk at every fill level, one score distribution each."""
    nh, nkv = LAYOUTS[q_per_kv]
    dist = ("random", "sharp", "flat")[(q_per_kv + hs // 64) % 3]
    run_case("b8_mixed", CASES["b8_mixed"](), nh, nkv, hs, dist, seed=100 * q_per_kv + hs)


@pytest.mark.parametrize("name,nh,nkv,hs,dist,log2_page", [
    ("b1_empty", 8, 8, 128, "random", None),
    ("b1_wrapped", 12, 4, 128, "sharp", None),
    ("b1_wrapped", 8, 2, 64, "flat", None),
    ("b8_to_wrap", 16, 2, 128, "flat", None),
    ("b8_to_wrap", 16, 4, 64, "random", 4),
    ("b8_mixed", 8, 4, 128, "sharp", 6),
    ("b64_tn2", 8, 4, 64, "random", None),
    ("b64_tn2", 12, 4, 128, "random", 4),
    ("ragged", 8, 4, 128, "random", None),
    ("ragged", 12, 4, 64, "sharp", None),
    ("ragged", 8, 1, 64, "flat", None),
    ("ragged", 12, 4, 128, "random", 4),
    ("ragged", 8, 8, 64, "sharp", 6),
    ("ragged_full", 16, 4, 128, "random", None),
    ("ragged_full", 8, 4, 64, "flat", None),
    ("ragged_full", 16, 2, 128, "random", 4),
    ("ragged_full", 12, 4, 64, "random", 6),
])
def test_chunks_row_maps_and_pages(name, nh, nkv, hs, dist, log2_page):
    """Prefill chunks at the callers' length limits, ragged row maps with padding rows, and the same launches through a
    page pool at RSTNET_KV_LOG2_PAGE_MIN (pages of 16) and at KV_PAGE (64)."""
    if log2_page is not None:
        assert log2_page in (_lib.KV_LOG2_PAGE_MIN, KV_PAGE.bit_length() - 1)
    run_case(name, CASES[name](), nh, nkv, hs, dist, seed=sum(map(ord, name)) + nh + hs, log2_page=log2_page)


@pytest.mark.parametrize("name,dist,log2_page,ostride", [
    ("moshi_start", "random", None, 1),
    ("moshi_wrap", "random", None, 1),
    ("moshi_wrap", "sharp", None, 1),
    ("moshi_10000", "random", None, 0),
    ("moshi_10000", "flat", None, 1),
    ("moshi_mixed", "random", None, 1),
    ("moshi_mixed", "sharp", 6, 1),
    ("moshi_mixed", "flat", 4, 1),
])
def test_moshi_scoring_window(name, dist, log2_page, ostride):
    """Moshi's non-streaming scope: rings of context + MAX_ROWS - 1 slots, 32 heads of 128 (MHA), 128-row chunks whose
    rows attend up to 3000 keys.  offset_stride 0 reads one counter for every row, as a one-stream scope may launch."""
    case = CASES[name]()
    assert case["cap"] - case["context"] + 1 == MAX_ROWS and sum(s >= 0 for s, _ in case["rows"]) == MAX_ROWS
    run_case(name, case, 32, 32, 128, dist, seed=sum(map(ord, name + dist)), log2_page=log2_page, ostride=ostride)


def test_chunk_lengths_reach_the_limits():
    """The chunk cases sit where the callers' limits bind: cap - context + 1 positions after the wrap (context < cap),
    cap - pos up to the wrap (context == cap), and MAX_ROWS in the Moshi scope."""
    assert len(CASES["b1_wrapped"]()["rows"]) == 160 - 40 + 1
    assert len(CASES["b8_mixed"]()["rows"]) == 8 * (72 - 64 + 1)
    assert len(CASES["b8_to_wrap"]()["rows"]) == 8 * (72 - 56)
    assert len(CASES["b64_tn2"]()["rows"]) == 64 * 2
    tns = lambda c: [sum(s == b for s, _ in c["rows"]) for b in range(c["B"])]
    assert tns(CASES["ragged"]()) == [20, 5, 100 - 92 + 1, 3, 100 - 92 + 1, 100 - 92 + 1]
    assert tns(CASES["ragged_full"]()) == [20, 5, 100 - 95, 1, 1, 1]
    assert tns(CASES["moshi_mixed"]()) == [50, 30, 48, 0, 0]


def test_bad_cap_or_context_fails_before_launch():
    """cap < 2 or context < 1 leaves every window empty: both entry points return an error and launch nothing.  The
    smallest legal ring (cap 2, context 1: each query attends its own key) returns that key's V exactly."""
    lib, st = _lib.lib(), ops._stream()
    B, nh, nkv, hs = 2, 4, 4, 64
    g = torch.Generator(device=DEV).manual_seed(3)
    q = torch.randn(B, nh * hs, generator=g, device=DEV).to(BF)
    kv = torch.randn(2, B, nkv, 2, hs, generator=g, device=DEV).to(BF)
    pool = torch.zeros(2, 2, nkv, 16, hs, dtype=BF, device=DEV)
    pt = torch.tensor([[0], [1]], dtype=torch.int32, device=DEV)
    offset = torch.tensor([3, 8], dtype=torch.int64, device=DEV)
    out = torch.zeros(B, nh * hs, dtype=BF, device=DEV)

    def both(cap, context):
        args = (q.data_ptr(), None, offset.data_ptr(), 1, None, None, out.data_ptr(), B, B, nh, nkv, hs, cap, context)
        return (lib.rstnet_lm_ring_decode_attention_bf16(*args[:1], kv.data_ptr(), *args[2:], st),
                lib.rstnet_lm_paged_decode_attention_bf16(*args[:1], pool.data_ptr(), *args[2:], pt.data_ptr(), 1, 4, st))

    n0 = _lib.launch_count()
    for cap, context in ((1, 1), (0, 1), (-3, 1), (2, 0), (4, -1)):
        ring_rc, paged_rc = both(cap, context)
        assert ring_rc != 0 and paged_rc != 0, (cap, context)
    assert _lib.launch_count() == n0
    _lib.check(lib.rstnet_lm_ring_decode_attention_bf16(q.data_ptr(), kv.data_ptr(), offset.data_ptr(), 1, None, None, out.data_ptr(),
                                                        B, B, nh, nkv, hs, 2, 1, st))
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0 + 1
    own = torch.stack([kv[1, b, :, int(offset[b]) % 2] for b in range(B)])     # [B, n_kv, hs]
    assert torch.equal(out.view(B, nh, hs), own)
