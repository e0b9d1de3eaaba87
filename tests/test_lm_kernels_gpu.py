"""Kernel-level GPU tests (-m gpu) of the LM decode path: the bf16 kernels behind include/rstnet_b200.h called through the
C ABI one by one, each compared element by element with an exact reference of the same operation on the same bf16
inputs: the oracle's own functions (oracle/lm_oracle.py, oracle/moshi_oracle.py) or a float64 evaluation.

Two tolerance classes:

* Bit-exact, where the kernel documents the eager roundings (elementwise kernels and copies): the embedding sum and
  gather, rotate-half RoPE and the K/V rows the launches append to their rings.  Outputs are compared with torch.equal
  (NaN == NaN where the contract poisons a row), and every ring slot a launch must not touch has to stay bit-identical.
  Two documented exceptions, both counted and reported: the Kyutai pair RoPE takes cos / sin from the GPU's cosf / sinf,
  which may differ from the CPU's in the last fp32 bit, so an element may differ by one bf16 ulp; the SiLU gating
  evaluates silu in fp32 with expf, so its bf16-rounded silu may land one bf16 ulp from the float64 one.
* Per-element bf16 bound, where there is a reduction (GEMMs, RMSNorm, attention):

      |out - ref64| <= ulp_bf16(ref64) + slack

  ref64 is the float64 result and ulp_bf16(x) the spacing of bf16 numbers at |x|.  GEMMs: slack = 2^-16 * S with S the
  float64 sum of |x_k * w_k| (+ |r|); fp32 accumulation over K <= 11008 terms stays far inside it, while a lost K chunk,
  a wrong K slice or a partial counted twice moves the result far outside.  Attention: slack = 2^-12 * max |v| over the
  attended keys.  Besides the bound, the fraction of outputs equal to bf16(ref64) is reported and held to a floor.

Every out-of-range case uses an input the kernels handle without reading the bad row: an embedding row with a bad id
reads no table row, and a position past the RoPE table reads table row 0.
"""
import math

import pytest
import torch

from oracle import lm_oracle as L
from oracle import moshi_oracle as M
from rstnet_b200 import _lib, ops
from rstnet_b200.lm import SkinnyGemm, interleave_gate_rows

pytestmark = pytest.mark.gpu
DEV, BF, F64 = "cuda", torch.bfloat16, torch.float64
NAN = float("nan")
SPLIT_CANDIDATES = (1, 2, 3, 4, 6, 8)   # the K split counts rstnet_skinny_gemm_create chooses from
GEMM_C = 2.0 ** -16
ATTN_C = 2.0 ** -12


# ------------------------------------------------------------------------------------------------------------- helpers
def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 numbers at |x| (float64): 2^(e-8) for |x| in [2^(e-1), 2^e), 2^-133 below the normal range."""
    x = x.to(F64)
    _, e = torch.frexp(x.abs())
    e = torch.where(x == 0, torch.full_like(e, -125), e.clamp(min=-125))
    return torch.pow(2.0, (e - 8).to(F64))


def check_bound(name, out, ref, slack, floor):
    """|out - ref| <= ulp_bf16(ref) + slack for every element and a bit-equal fraction (out == bf16(ref)) >= floor.
    Prints the worst error in bf16 ulps of ref and the bit-equal fraction."""
    out = out.detach().to("cpu", F64)
    ref = ref.detach().to("cpu", F64)
    slack = slack.detach().to("cpu", F64) if torch.is_tensor(slack) else torch.tensor(float(slack), dtype=F64)
    err = (out - ref).abs()
    u = ulp_bf16(ref)
    bad = ~(err <= u + slack)                       # NaN counts as outside
    worst = float(torch.nan_to_num(err / u, nan=float("inf")).max())
    used = float(torch.nan_to_num(err / (u + slack), nan=float("inf")).max())
    eq = float((out == ref.to(BF).to(F64)).to(F64).mean())
    print(f"[lm-kernels] {name}: worst {worst:.3f} bf16 ulps ({used:.3f} of the bound), bit-equal {eq:.5f} of {out.numel()}")
    if bad.any():
        i = tuple(int(v) for v in bad.nonzero()[0])
        sl = slack.expand_as(ref)[i] if slack.dim() else slack
        raise AssertionError(f"{name}: {int(bad.sum())}/{out.numel()} elements outside ulp + slack; first at {i}: "
                             f"out {float(out[i])!r} ref {float(ref[i])!r} ulp {float(u[i])!r} slack {float(sl)!r}")
    assert eq >= floor, f"{name}: only {eq:.5f} of the outputs equal bf16(ref64) (floor {floor})"
    return worst, eq


def same(a: torch.Tensor, b: torch.Tensor) -> bool:
    """torch.equal that also takes NaN == NaN (the poisoned rows of the out-of-range contract)."""
    a, b = a.cpu(), b.cpu()
    return a.shape == b.shape and a.dtype == b.dtype and bool(((a == b) | (a.isnan() & b.isnan())).all())


def error_flags(clear: bool) -> int:
    """rstnet_device_error_flags: bit 0 (1) id out of range, bit 1 (2) RoPE position past the table.  The word is
    process-global, so every test that reads it clears it first."""
    return int(_lib.lib().rstnet_device_error_flags(int(clear)))


def gemm_ref(x: torch.Tensor, w: torch.Tensor, r=None):
    """float64 x @ w^T (+ r) and S = |x| @ |w|^T (+ |r|) of bf16 operands."""
    x, w = x.to(F64), w.to(F64)
    ref, s = x @ w.t(), x.abs() @ w.abs().t()
    if r is not None:
        ref, s = ref + r.to(F64), s + r.to(F64).abs()
    return ref, s


def k_slices_written(ws: torch.Tensor, M: int, N: int, max_splits: int) -> int:
    """K slices that wrote fp32 partials into a workspace that was all NaN before the run: slices 0..n-1 must be
    written completely and the rest not at all.  0 = one slice that wrote `out` directly."""
    w = ~ws[:max_splits * M * N].view(max_splits, M * N).isnan()
    full = w.all(1)
    n = int(full.sum())
    assert bool(full[:n].all()) and not bool(w[n:].any()), "K slices written incompletely or out of order"
    return n


def forced_splits(N: int, K: int, max_splits: int) -> int:
    """The K split count rstnet_skinny_gemm_create must choose.  With few 128-row N tiles it wants 1.5 CTAs per SM, more
    than 8 slices, so it takes the largest candidate <= max_splits that leaves every slice >= 8 of the K/64 chunks.
    Split-K needs N % 4 == 0."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert 1.5 * sms / -(-N // 128) >= 8, f"N = {N} has too many tiles for the split count to be forced on {sms} SMs"
    if N % 4:
        return 1
    return max(c for c in SPLIT_CANDIDATES if c <= max_splits and (c == 1 or (K // 64) // c >= 8))


def ring_keys(pos: int, cap: int, context: int) -> torch.Tensor:
    """Slots a query at position `pos` attends once its own key is in the ring: the labels of RingKVCache.complete
    (the oracle's L.Ring) under the mask (pos_k >= 0) & (delta >= 0) & (delta < context)."""
    ring = L.Ring(1, 1, 1, cap, torch.float32)
    ring.end_offset = pos
    z = torch.zeros(1, 1, 1, 1)
    _, _, pk = ring.complete(z, z)
    delta = pos - pk
    return ((pk >= 0) & (delta >= 0) & (delta < context)).nonzero()[:, 0]


def softmax_attention64(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float) -> torch.Tensor:
    """float64 softmax(q k^T * scale) v; q [..., nq, hs], k / v [..., nk, hs]."""
    s = torch.einsum("...qd,...kd->...qk", q.to(F64), k.to(F64)) * scale
    return torch.einsum("...qk,...kd->...qd", torch.softmax(s, -1), v.to(F64))


def _randn(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(BF)


# ------------------------------------------------------------------------------ skinny GEMM, fused residual + RMSNorm
@pytest.mark.parametrize("M,N,K,max_splits,kyutai,spread", [
    (1, 144, 1024, 1, False, False),
    (1, 4096, 4288, 8, True, False),
    (64, 256, 4288, 3, False, True),
    (64, 1024, 1024, 1, True, True),
    (64, 4096, 4288, 4, False, False),
    (128, 144, 4288, 6, True, True),
    (128, 1024, 4288, 8, False, True),
    (128, 4096, 1024, 1, True, False),
])
def test_skinny_gemm_residual_rmsnorm_finalize(M, N, K, max_splits, kyutai, spread):
    """fin_mode 1: out = bf16(X W^T + R) in place on the residual stream (R aliases out, as lm.py runs it) and
    aux = RMSNorm(out) * w across the 4-CTA cluster, lit (eps inside the rsqrt after the mean) and Kyutai form.  `spread`
    scales the rows 2^-8 .. 2^8 apart, so a row mix-up or a slice sum taken from the wrong row cannot hide."""
    g = torch.Generator().manual_seed(1000 * M + N + K)
    x, r = torch.randn(M, K, generator=g), torch.randn(M, N, generator=g)
    if spread:
        s = 4.0 ** (torch.arange(M) % 9 - 4).float()[:, None]
        x, r = x * s, r * s
    x, r = x.to(BF), r.to(BF)
    w = _randn(g, N, K, scale=K ** -0.5)
    nw = (1 + 0.1 * torch.randn(N, generator=g)).to(BF)
    eps = 1e-8 if kyutai else 1e-5
    out = r.to(DEV)
    aux = torch.full((M, N), NAN, dtype=BF, device=DEV)
    ws = torch.full((max_splits * M * N,), NAN, dtype=torch.float32, device=DEV)
    SkinnyGemm(x.to(DEV), w.to(DEV), out, out, ws, max_splits=max_splits, norm_w=nw.to(DEV), aux=aux, eps=eps,
               kyutai=kyutai).run()
    torch.cuda.synchronize()
    n = k_slices_written(ws, M, N, max_splits)
    assert n >= 1 and (n == 1) == (max_splits == 1), n
    ref, S = gemm_ref(x, w, r)
    check_bound(f"skinny fin_mode 1 out M {M} N {N} K {K} splits {n}", out, ref, GEMM_C * S, 0.99)
    # aux against the float64 RMSNorm of the kernel's own stored out, with L.rms_norm / L.rms_norm_f32's eps placement and
    # multiplication order
    o, nw64 = out.cpu().to(F64), nw.to(F64)
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    ms = (o * o).mean(-1, keepdim=True)
    y = o * (nw64 * torch.rsqrt(eps32 + ms)) if kyutai else (o * torch.rsqrt(ms + eps32)) * nw64
    check_bound(f"skinny fin_mode 1 aux ({'kyutai' if kyutai else 'lit'}) M {M} N {N}", aux, y, 0.0, 0.999)


# ---------------------------------------------------------------------------------------------- standalone RMSNorm
@pytest.mark.parametrize("kyutai", [False, True])
@pytest.mark.parametrize("rows", [1, 37, 256])
@pytest.mark.parametrize("dim", [1000, 1024, 2048, 3072, 4096])
def test_rms_norm_per_element(dim, rows, kyutai):
    """rstnet_lm_rms_norm_bf16 (the first pre-norm of every frame, on the residual stream) vs the float64 RMSNorm with the
    aux check's eps placement and multiplication order, one bf16 ulp and no slack.  Rows are scaled 2^-8 .. 2^8 apart
    and the last of several rows is all zero, so a row mix-up or a sum taken over the wrong row cannot hide; dim 1000 is
    not a multiple of the 256-thread block."""
    g = torch.Generator().manual_seed(dim + rows + kyutai)
    s = 2.0 ** (torch.arange(rows) % 17 - 8).float()[:, None]
    x = (torch.randn(rows, dim, generator=g) * s).to(BF)
    if rows > 1:
        x[-1] = 0
    w = (1 + 0.1 * torch.randn(dim, generator=g)).to(BF)
    eps = 1e-8 if kyutai else 1e-5
    y = torch.full((rows + 1, dim), NAN, dtype=BF, device=DEV)   # one row past the output must stay untouched
    xd, wd = x.to(DEV), w.to(DEV)
    _lib.check(_lib.lib().rstnet_lm_rms_norm_bf16(xd.data_ptr(), wd.data_ptr(), y.data_ptr(), rows, dim, eps, int(kyutai),
                                                  ops._stream()))
    torch.cuda.synchronize()
    assert y[rows].isnan().all()
    o, w64 = x.to(F64), w.to(F64)
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    ms = (o * o).mean(-1, keepdim=True)
    ref = o * (w64 * torch.rsqrt(eps32 + ms)) if kyutai else (o * torch.rsqrt(ms + eps32)) * w64
    check_bound(f"rms norm ({'kyutai' if kyutai else 'lit'}) rows {rows} dim {dim}", y[:rows], ref, 0.0, 0.999)
    if rows > 1:
        assert bool((y[rows - 1] == 0).all()), "an all-zero row normalises to zeros"


# --------------------------------------------------------------------------------- skinny GEMM, SiLU gating (2 and 3)
def _gating_chain(a: torch.Tensor, b: torch.Tensor):
    """The documented roundings of the gating, evaluated in float64: bf16(bf16(silu(bf16(a))) * bf16(b)).  Also returns
    the one-ulp-of-silu allowance: the kernels evaluate silu in fp32 with expf, which may put it on the other side of a
    bf16 rounding boundary."""
    a64, b64 = a.to(BF).to(F64), b.to(BF).to(F64)
    s = (a64 / (1.0 + torch.exp(-a64))).to(BF).to(F64)
    ref = (s * b64).to(BF).to(F64)          # s * b is exact in float64 (two 8-bit significands)
    return ref, b64.abs() * ulp_bf16(s)


def _check_gating(name, out, a, b):
    ref, tol = _gating_chain(a, b)
    out64 = out.cpu().to(F64)
    err = (out64 - ref).abs()
    off = int((out64 != ref).sum())
    print(f"[lm-kernels] {name}: {off}/{out.numel()} outputs differ from the float64 rounding chain")
    assert bool((err <= ulp_bf16(ref) + tol).all()), f"{name}: worst error {float(err.max())}"
    assert off <= 1e-3 * out.numel() + 1, f"{name}: {off} outputs differ from the rounding chain"


@pytest.mark.parametrize("M,K,I,max_splits", [(5, 256, 96, 8), (17, 4288, 96, 8), (64, 1024, 682, 8), (128, 512, 682, 1),
                                              (64, 4288, 682, 3), (33, 4288, 1000, 6)])
def test_skinny_gemm_silu_gating_finalize_and_epilogue(M, K, I, max_splits):
    """fin_mode 2 (finalize kernel over the stacked [gate; value] weight) and fin_mode 3 (in-epilogue gating over the
    row-interleaved weight).  The GEMM sums (the fp32 partials mode 2 leaves in its workspace) are held to the GEMM bound;
    the gated outputs to the float64 rounding chain of those sums; mode 3 and mode 2 with one K slice accumulate the same
    products in the same order and must agree bit for bit.  I = 96 and 682 leave a partial 128-row weight tile."""
    g = torch.Generator().manual_seed(M + K + I)
    N = 2 * I
    x = _randn(g, M, K)
    w1, w2 = _randn(g, I, K, scale=K ** -0.5), _randn(g, I, K, scale=K ** -0.5)
    xd, stacked = x.to(DEV), torch.cat([w1, w2], 0).to(DEV).contiguous()
    outs, sums = {}, {}
    for c in (max_splits, 1):
        ws = torch.full((c * M * N,), NAN, dtype=torch.float32, device=DEV)
        o = torch.full((M, I), NAN, dtype=BF, device=DEV)
        SkinnyGemm(xd, stacked, None, None, ws, max_splits=c, silu_out=o).run()
        torch.cuda.synchronize()
        n = k_slices_written(ws, M, N, c)
        assert n == forced_splits(N, K, c), (c, n)
        part = ws[:n * M * N].view(n, M, N).cpu()
        acc = part[0].clone()
        for s in range(1, n):            # the finalize kernel's order: slice 0 + slice 1 + ... in fp32
            acc += part[s]
        outs[c], sums[c] = o, acc
    o3 = torch.full((M, I), NAN, dtype=BF, device=DEV)
    SkinnyGemm(xd, interleave_gate_rows(w1.to(DEV), w2.to(DEV)), None, None, None, silu_out=o3, interleaved=True).run()
    torch.cuda.synchronize()
    ref_a, s_a = gemm_ref(x, w1)
    ref_b, s_b = gemm_ref(x, w2)
    for c, acc in sums.items():
        for half, ref, S in ((acc[:, :I], ref_a, s_a), (acc[:, I:], ref_b, s_b)):
            err = (half.to(F64) - ref).abs()
            assert bool((err <= GEMM_C * S).all()), (c, float((err / S).max()))
        _check_gating(f"skinny fin_mode 2 M {M} K {K} I {I} splits {forced_splits(N, K, c)}", outs[c], acc[:, :I], acc[:, I:])
    assert torch.equal(o3, outs[1]), "in-epilogue gating (fin_mode 3) != finalize gating (fin_mode 2) with one K slice"
    if forced_splits(N, K, max_splits) == 1:
        assert torch.equal(o3, outs[max_splits])
    ref, _ = _gating_chain(ref_a, ref_b)
    eq = float((o3.cpu().to(F64) == ref).to(F64).mean())
    print(f"[lm-kernels] skinny fin_mode 3 M {M} K {K} I {I}: bit-equal to the chain of the float64 sums {eq:.5f}")
    assert eq >= 0.98


# ------------------------------------------------------------------------------------------------------- embeddings
def _table(g, rows, E):
    # rows of very different magnitude, so that the bf16 rounding after every add of the sum matters
    return (torch.randn(rows, E, generator=g) * 4.0 ** torch.randint(-3, 4, (rows, 1), generator=g)).to(BF)


def test_embed_sum_bit_exact_and_bad_ids():
    """rstnet_lm_embed_sum_bf16 == L.embed_sum bit for bit (n_q = 8, seq_stride 12 > n_q + 1): ids -1 (zero row), 0 and
    rows - 1 in every table, text id -1 as a zero row too.  A row with ids -2 and `rows` is all NaN, the other rows stay
    exact and error bit 0 is set until cleared."""
    lib, st = _lib.lib(), ops._stream()
    g = torch.Generator().manual_seed(31)
    n_q, E, B, stride, wte_rows, rows = 8, 320, 6, 12, 50, 33
    wte, tables = _table(g, wte_rows, E), [_table(g, rows, E) for _ in range(n_q)]
    seq = torch.full((B, stride), 10 ** 9, dtype=torch.int64)    # columns past n_q + 1 are not ids and must not be read
    seq[:, 0] = torch.randint(0, wte_rows, (B,), generator=g)
    seq[:, 1:n_q + 1] = torch.randint(-1, rows, (B, n_q), generator=g)
    seq[0, 1:n_q + 1] = -1
    seq[1, :n_q + 1] = 0
    seq[2, 0], seq[2, 1:n_q + 1] = wte_rows - 1, rows - 1
    seq[3, 0] = -1
    w = {f"input_emb.{cb}.weight": tables[cb] for cb in range(n_q)}
    w["transformer.wte.weight"] = torch.cat([wte, torch.zeros(1, E, dtype=BF)])   # row wte_rows: the zero row of text id -1
    ids = seq[:, :n_q + 1].clone()
    ids[:, 0] = torch.where(ids[:, 0] == -1, wte_rows, ids[:, 0])
    ref = L.embed_sum(ids, w, L.SMALL)
    assert L.SMALL.n_q == n_q
    wte_d, tabs_d = wte.to(DEV), [t.to(DEV) for t in tables]
    ptrs = torch.tensor([t.data_ptr() for t in tabs_d], dtype=torch.int64, device=DEV)

    def run(s):
        x = torch.full((B, E), NAN, dtype=BF, device=DEV)
        sd = s.to(DEV)
        _lib.check(lib.rstnet_lm_embed_sum_bf16(sd.data_ptr(), stride, wte_d.data_ptr(), wte_rows, ptrs.data_ptr(), rows, n_q, E,
                                                x.data_ptr(), B, st))
        return x.cpu()

    error_flags(True)
    assert torch.equal(run(seq), ref)
    assert error_flags(False) == 0
    bad = seq.clone()
    bad[4, 3], bad[4, 0], bad[4, 6] = -2, wte_rows, rows
    x = run(bad)
    assert x[4].isnan().all()
    keep = torch.arange(B) != 4
    assert torch.equal(x[keep], ref[keep])
    assert error_flags(True) == 1
    assert error_flags(False) == 0


def test_embed_rows_bit_exact_and_bad_ids():
    """rstnet_lm_embed_rows_bf16 with id_stride 3 == L.scaled_embedding (zero row for -1, rows 0 and rows - 1); ids -2
    and `rows` give NaN rows and error bit 0, the other rows stay exact."""
    lib, st = _lib.lib(), ops._stream()
    g = torch.Generator().manual_seed(32)
    D, rows, R, id_stride = 192, 40, 7, 3
    table = _table(g, rows, D)
    ids = torch.full((R, id_stride), 10 ** 9, dtype=torch.int64)
    ids[:, 0] = torch.randint(-1, rows, (R,), generator=g)
    ids[0, 0], ids[1, 0], ids[2, 0] = -1, 0, rows - 1
    ref = L.scaled_embedding(ids[:, 0], table)
    td = table.to(DEV)

    def run(i):
        out = torch.full((R, D), NAN, dtype=BF, device=DEV)
        idd = i.to(DEV)
        _lib.check(lib.rstnet_lm_embed_rows_bf16(idd.data_ptr(), id_stride, td.data_ptr(), rows, D, out.data_ptr(), R, st))
        return out.cpu()

    error_flags(True)
    assert torch.equal(run(ids), ref)
    assert error_flags(False) == 0
    bad = ids.clone()
    bad[3, 0], bad[5, 0] = -2, rows
    out = run(bad)
    keep = torch.ones(R, dtype=torch.bool)
    keep[[3, 5]] = False
    assert out[~keep].isnan().all() and torch.equal(out[keep], ref[keep])
    assert error_flags(True) == 1
    assert error_flags(False) == 0


# ------------------------------------------------------------------------------------- rotate-half RoPE + ring append
def _rope_append(nh, nkv, hs, rope_n, offsets, Tn, cap, rope_rows, seed):
    """One rstnet_lm_rope_kv_append_bf16 launch over Tn time-major rows per stream (per-stream offsets) into a ring full
    of random values; returns (q_out, kv, expected q_out, expected kv, bad) with the expectation from L.split_qkv +
    L.rope_partial on tables long enough for every position, and bad[tl, b] = the position is >= rope_rows."""
    B = len(offsets)
    cfg = L.LMConfig(n_head=nh, n_query_groups=nkv, head_size=hs, rotary_percentage=rope_n / hs,
                     block_size=max(offsets) + Tn)
    assert cfg.rope_n_elem == rope_n
    cos, sin = L.rope_cache(cfg, BF)
    g = torch.Generator().manual_seed(seed)
    qkv = _randn(g, Tn * B, (nh + 2 * nkv) * hs)
    kv0 = _randn(g, 2, B, nkv, cap, hs)
    off = torch.tensor(offsets, dtype=torch.int64)
    q_out = torch.full((Tn * B, nh * hs), NAN, dtype=BF, device=DEV)
    kv = kv0.to(DEV)
    qkv_d, cos_d, sin_d, off_d = qkv.to(DEV), cos.to(DEV), sin.to(DEV), off.to(DEV)
    _lib.check(_lib.lib().rstnet_lm_rope_kv_append_bf16(qkv_d.data_ptr(), cos_d.data_ptr(), sin_d.data_ptr(), rope_rows, rope_n,
                                                        off_d.data_ptr(), 1, None, None, q_out.data_ptr(), kv.data_ptr(), Tn * B, B,
                                                        nh, nkv, hs, cap, ops._stream()))
    torch.cuda.synchronize()
    # row tl * B + b is stream b at position offsets[b] + tl
    q, k, v = L.split_qkv(qkv.view(Tn, B, -1).transpose(0, 1).contiguous(), cfg)     # [B, heads, Tn, hs]
    k, v = [t.reshape(B, nkv, -1, Tn, hs)[:, :, 0] for t in (k, v)]                  # K/V once per group
    q_exp = torch.empty(Tn, B, nh, hs, dtype=BF)
    kv_exp = kv0.clone()
    bad = torch.zeros(Tn, B, dtype=torch.bool)
    for b in range(B):
        pos = offsets[b] + torch.arange(Tn)
        qr = L.rope_partial(q[b:b + 1], cos[pos], sin[pos], rope_n)[0]
        kr = L.rope_partial(k[b:b + 1], cos[pos], sin[pos], rope_n)[0]
        for tl in range(Tn):
            p = int(pos[tl])
            qo, ko = qr[:, tl].clone(), kr[:, tl].clone()
            if p >= rope_rows:
                bad[tl, b] = True
                qo[:, :rope_n], ko[:, :rope_n] = NAN, NAN
            q_exp[tl, b] = qo
            kv_exp[0, b, :, p % cap], kv_exp[1, b, :, p % cap] = ko, v[b, :, tl]
    return q_out.cpu(), kv.cpu(), q_exp.view(Tn * B, nh * hs), kv_exp, bad


@pytest.mark.parametrize("rope_div", [1, 2, 4])
@pytest.mark.parametrize("nh,nkv,hs", [(4, 4, 128), (4, 2, 64), (6, 2, 128), (8, 1, 64)])
def test_rope_kv_append_gqa_partial_rotary_per_stream(nh, nkv, hs, rope_div):
    """MHA, GQA (even and odd q_per_kv), MQA; rotary over hs, hs/2, hs/4 dims; per-stream offsets at different fill
    levels (empty, partial, wrapping inside the launch, wrapped) with 3 prefill rows per stream.  q and every ring slot
    bit-exact, untouched slots unchanged."""
    cap = 16
    error_flags(True)
    q, kv, q_exp, kv_exp, bad = _rope_append(nh, nkv, hs, hs // rope_div, [0, 5, cap - 2, 2 * cap + 3], 3, cap, 64,
                                             seed=nh * 100 + nkv * 10 + rope_div)
    assert not bad.any()
    assert torch.equal(q, q_exp), "rotated q must match L.rope_partial bit for bit"
    assert torch.equal(kv, kv_exp), "ring contents must match bit for bit (appended rows and untouched slots)"
    assert error_flags(False) == 0


def test_rope_kv_append_position_past_table_poisons_only_that_row():
    """A position >= rope_rows: that row's rotated q / k dims are NaN (the pass-through dims and v are still copied), every
    other row is exact and error bit 1 is set.  Stream 1 crosses the end of the table inside the launch, stream 2 lies
    past it."""
    rope_rows = 40
    error_flags(True)
    q, kv, q_exp, kv_exp, bad = _rope_append(6, 2, 128, 64, [2, rope_rows - 2, rope_rows + 5], 3, 16, rope_rows, seed=7)
    assert int(bad.sum()) == 4 and bool(bad[2, 1]) and not bool(bad[:2, 1].any())
    assert same(q, q_exp) and same(kv, kv_exp)
    assert q.view(3, 3, -1)[~bad].isnan().sum() == 0
    assert error_flags(True) == 2
    assert error_flags(False) == 0


# ------------------------------------------------------------------------------------------- Kyutai pair RoPE + append
@pytest.mark.parametrize("hd", [64, 128])
def test_rope_pair_kv_append_large_offsets(hd):
    """rstnet_lm_rope_pair_kv_append_bf16 vs M.rope_pairs with per-stream offsets up to ~50,000 (an hour of 12.5 Hz frames,
    where the fp32 angle freqs * t is large) and 3 rows per stream: within one bf16 ulp where the GPU's cosf / sinf and the
    CPU's differ in the last fp32 bit (counted), v and every untouched ring slot exact."""
    B, H, Tn, cap, max_period = 4, 4, 3, 16, 10000.0
    offsets = [0, 7, 12345, 49998]
    g = torch.Generator().manual_seed(hd)
    qkv = _randn(g, Tn * B, 3, H, hd)
    kv0 = _randn(g, 2, B, H, cap, hd)
    # freqs as rstnet_b200/moshi.py passes them (modules/rope.py:35-36)
    freqs = torch.exp(torch.arange(hd // 2, dtype=torch.float32) * (-math.log(max_period) * 2 / hd))
    q_out = torch.full((Tn * B, H * hd), NAN, dtype=BF, device=DEV)
    kv = kv0.to(DEV)
    qkv_d, off_d, fr_d = qkv.to(DEV), torch.tensor(offsets, device=DEV), freqs.to(DEV)
    _lib.check(_lib.lib().rstnet_lm_rope_pair_kv_append_bf16(qkv_d.data_ptr(), off_d.data_ptr(), 1, q_out.data_ptr(), kv.data_ptr(),
                                                             Tn * B, B, H, hd, cap, fr_d.data_ptr(), ops._stream()))
    torch.cuda.synchronize()
    x = qkv.view(Tn, B, 3, H, hd)
    q_exp = torch.empty(Tn, B, H, hd, dtype=BF)
    kv_exp, tol = kv0.clone(), torch.zeros(2, B, H, cap, hd, dtype=F64)
    for b in range(B):
        qb, kb = [x[:, b, i].permute(1, 0, 2).contiguous()[None] for i in (0, 1)]     # [1, H, Tn, hd]
        qo, ko = M.rope_pairs(qb, kb, offsets[b], max_period)
        for tl in range(Tn):
            slot = (offsets[b] + tl) % cap
            q_exp[tl, b] = qo[0, :, tl]
            kv_exp[0, b, :, slot], kv_exp[1, b, :, slot] = ko[0, :, tl], x[tl, b, 2]
            tol[0, b, :, slot] = ulp_bf16(ko[0, :, tl])
    q_exp = q_exp.view(Tn * B, H * hd)
    q, kv = q_out.cpu(), kv.cpu()
    dq, dk = (q.to(F64) - q_exp.to(F64)).abs(), (kv.to(F64) - kv_exp.to(F64)).abs()
    print(f"[lm-kernels] pair RoPE hd {hd}: {int((dq > 0).sum())}/{q.numel()} q and {int((dk > 0).sum())}/{int((tol > 0).sum())} "
          f"appended k elements one bf16 ulp off (cosf / sinf vs the CPU's cos / sin)")
    assert bool((dq <= ulp_bf16(q_exp)).all()) and bool((dk <= tol).all())
    assert int((dq > 0).sum()) <= 1e-2 * q.numel()


# --------------------------------------------------------------------------------------------- depth attention
@pytest.mark.parametrize("quirk", [1, 0])
@pytest.mark.parametrize("hd", [32, 64, 128])
@pytest.mark.parametrize("cap", [2, 4, 8])
def test_depth_attention_every_step(cap, hd, quirk):
    """rstnet_lm_depth_attention_bf16 at every step 0..cap-1: K/V rows bit-exact at slot `step` (other slots unchanged) and
    the output vs a float64 softmax over the keys L.Ring.complete leaves attendable (ring_quirk 1: the streaming form,
    which masks key 0 on the last step) or over keys 0..step (ring_quirk 0: KVCacheResult.from_kv)."""
    lib, st = _lib.lib(), ops._stream()
    B, H = 3, 4
    g = torch.Generator().manual_seed(cap * 1000 + hd * 10 + quirk)
    kv_exp = _randn(g, 2, B, H, cap, hd)
    kvd = kv_exp.to(DEV)
    ring = L.Ring(1, 1, 1, cap, torch.float32)
    z = torch.zeros(1, 1, 1, 1)
    for step in range(cap):
        qkv = _randn(g, B, 3, H, hd)
        out = torch.full((B, H * hd), NAN, dtype=BF, device=DEV)
        qd = qkv.to(DEV)
        _lib.check(lib.rstnet_lm_depth_attention_bf16(qd.data_ptr(), kvd.data_ptr(), out.data_ptr(), B, H, hd, cap, step, quirk, st))
        torch.cuda.synchronize()
        kv_exp[0, :, :, step], kv_exp[1, :, :, step] = qkv[:, 1], qkv[:, 2]
        assert torch.equal(kvd.cpu(), kv_exp), step
        _, _, pk = ring.complete(z, z)
        keys = ((pk >= 0) & (step - pk >= 0)).nonzero()[:, 0] if quirk else torch.arange(step + 1)
        if quirk and step == cap - 1:
            assert 0 not in keys.tolist()
        k_, v_ = kv_exp[0][:, :, keys], kv_exp[1][:, :, keys]
        ref = softmax_attention64(qkv[:, 0][:, :, None], k_, v_, hd ** -0.5)[:, :, 0]
        slack = ATTN_C * v_.to(F64).abs().amax((2, 3))[:, :, None]
        check_bound(f"depth attention cap {cap} hd {hd} quirk {quirk} step {step}", out.view(B, H, hd), ref, slack, 0.98)
