"""GPU tests (-m gpu) of decode scopes wider than 128 streams: the 256-column instantiation of the weight-streaming GEMM
(129 <= M <= 256, two consumer warpgroups that each own one 64-row half of the weight tile) through every fused finalize
and split count, and the LM, the Moshi twin and the duplex engine at 256 streams.

The GEMM checks use the per-element bound of test_lm_kernels_gpu.py, |out - ref64| <= ulp_bf16(ref64) + 2^-16 * S.  Rows m
and m + 128 are scaled apart, so output written to the other half of the streams cannot stay inside it.  Outputs and
workspaces are NaN-filled before a run: the split count that ran is read from the workspace, and a NaN canary after each
output must survive.
"""
import dataclasses

import pytest
import torch

import test_lm_kernels_gpu as KT
from oracle import lm_oracle as L
from oracle import moshi_oracle as MO
from rstnet_b200._lib import RstnetError
from rstnet_b200.lm import GPT, MAX_STREAMS, Config, SkinnyGemm, interleave_gate_rows

pytestmark = pytest.mark.gpu
DEV, BF, F64 = "cuda", torch.bfloat16, torch.float64
NAN = float("nan")
CANARY = 64


def _rows(g, M, K, scale=1.0):
    """[M, K] bf16 rows; rows 128..255 are 3x rows 0..127, so a stream-half mix-up changes a result by far more than the
    bound."""
    x = torch.randn(M, K, generator=g) * scale
    x[128:] *= 3.0
    return x.to(BF)


def _nan_out(M, N):
    """An [M, N] bf16 output view followed by CANARY NaNs in the same allocation."""
    buf = torch.full((M * N + CANARY,), NAN, dtype=BF, device=DEV)
    return buf, buf[:M * N].view(M, N)


def _canary_ok(buf, M, N):
    assert bool(buf[M * N:].isnan().all()), "the GEMM wrote past the end of its output"


def expected_splits(M, N, K, max_splits):
    """The K split count rstnet_skinny_gemm_create must choose.  M <= 128: the rule test_lm_kernels_gpu.forced_splits
    states.  M > 128 (one CTA per SM): the largest candidate <= max_splits that leaves every slice >= 8 of the K/64 chunks
    and keeps all n_tiles * splits CTAs in one wave."""
    if M <= 128:
        return KT.forced_splits(N, K, max_splits)
    if N % 4:
        return 1
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = -(-N // 128)
    return max(c for c in KT.SPLIT_CANDIDATES
               if c <= max_splits and (c == 1 or ((K // 64) // c >= 8 and c * tiles <= sms)))


# ------------------------------------------------------------------------------- skinny GEMM, plain and residual
@pytest.mark.parametrize("M,N,K,res,max_splits", [
    (129, 256, 4288, True, 8),     # 67 K chunks: 8 slices of 9, the last 4
    (136, 1000, 1024, False, 1),
    (200, 384, 2112, True, 2),     # 33 chunks: 17 + 16
    (255, 130, 1088, True, 4),     # N % 4 != 0: no split-K
    (256, 512, 4160, True, 4),     # 65 chunks: 17, 17, 17, 14
    (256, 3072, 4288, False, 8),   # 24 tiles: 4 splits, the most that fit one wave of CTAs
    (200, 1536, 1024, False, 8),   # 16 chunks: at most 2 slices of >= 8
    (129, 77, 512, False, 8),      # N % 4 != 0, a partial 128-row weight tile
])
def test_wide_skinny_gemm_plain(M, N, K, res, max_splits):
    g = torch.Generator().manual_seed(7 * M + N + K)
    x = _rows(g, M, K)
    w = KT._randn(g, N, K, scale=K ** -0.5)
    r = _rows(g, M, N) if res else None
    buf, out = _nan_out(M, N)
    ws = torch.full((max_splits * M * N,), NAN, dtype=torch.float32, device=DEV)
    SkinnyGemm(x.to(DEV), w.to(DEV), out, None if r is None else r.to(DEV), ws, max_splits=max_splits).run()
    torch.cuda.synchronize()
    n = KT.k_slices_written(ws, M, N, max_splits) if N % 4 == 0 else 0
    want = expected_splits(M, N, K, max_splits)
    assert max(n, 1) == want, (n, want)
    _canary_ok(buf, M, N)
    ref, S = KT.gemm_ref(x, w, r)
    KT.check_bound(f"wide skinny M {M} N {N} K {K} res {res} splits {max(n, 1)}", out, ref, KT.GEMM_C * S, 0.99)


# ------------------------------------------------------------------------- skinny GEMM, residual + RMSNorm finalize
@pytest.mark.parametrize("M,N,K,max_splits,kyutai", [
    (129, 1024, 4288, 8, False),
    (256, 3072, 1024, 2, True),
    (255, 144, 4288, 4, True),
    (136, 256, 2112, 1, False),
    (256, 2048, 4288, 8, True),
    (200, 1024, 4160, 6, False),
])
def test_wide_skinny_gemm_residual_rmsnorm_finalize(M, N, K, max_splits, kyutai):
    """fin_mode 1 in place on the residual stream, lit and Kyutai RMSNorm of the stored result (as
    test_lm_kernels_gpu.test_skinny_gemm_residual_rmsnorm_finalize); the cluster finalize runs M x 4 CTAs."""
    g = torch.Generator().manual_seed(1000 * M + N + K)
    x, r = _rows(g, M, K), _rows(g, M, N)
    w = KT._randn(g, N, K, scale=K ** -0.5)
    nw = (1 + 0.1 * torch.randn(N, generator=g)).to(BF)
    eps = 1e-8 if kyutai else 1e-5
    out = r.to(DEV)
    abuf, aux = _nan_out(M, N)
    ws = torch.full((max_splits * M * N,), NAN, dtype=torch.float32, device=DEV)
    SkinnyGemm(x.to(DEV), w.to(DEV), out, out, ws, max_splits=max_splits, norm_w=nw.to(DEV), aux=aux, eps=eps,
               kyutai=kyutai).run()
    torch.cuda.synchronize()
    n = KT.k_slices_written(ws, M, N, max_splits)
    assert n == expected_splits(M, N, K, max_splits), n
    _canary_ok(abuf, M, N)
    ref, S = KT.gemm_ref(x, w, r)
    KT.check_bound(f"wide fin_mode 1 out M {M} N {N} K {K} splits {n}", out, ref, KT.GEMM_C * S, 0.99)
    o, nw64 = out.cpu().to(F64), nw.to(F64)
    eps32 = float(torch.tensor(eps, dtype=torch.float32))
    ms = (o * o).mean(-1, keepdim=True)
    y = o * (nw64 * torch.rsqrt(eps32 + ms)) if kyutai else (o * torch.rsqrt(ms + eps32)) * nw64
    KT.check_bound(f"wide fin_mode 1 aux ({'kyutai' if kyutai else 'lit'}) M {M} N {N}", aux, y, 0.0, 0.999)


# ------------------------------------------------------------------------------------ skinny GEMM, SiLU gating 2 and 3
@pytest.mark.parametrize("M,K,I,max_splits", [(129, 1024, 682, 8), (256, 4288, 96, 4), (200, 512, 1000, 2),
                                              (256, 1024, 682, 1), (255, 4288, 682, 8)])
def test_wide_skinny_gemm_silu_gating(M, K, I, max_splits):
    """fin_mode 2 (stacked [gate; value], finalize kernel) and fin_mode 3 (row-interleaved weight, gating in the
    epilogue, one shuffle inside a warp) under the documented roundings; with one K slice the two agree bit for bit."""
    g = torch.Generator().manual_seed(M + K + I)
    N = 2 * I
    x = _rows(g, M, K)
    w1, w2 = KT._randn(g, I, K, scale=K ** -0.5), KT._randn(g, I, K, scale=K ** -0.5)
    xd, stacked = x.to(DEV), torch.cat([w1, w2], 0).to(DEV).contiguous()
    outs, sums = {}, {}
    for c in (max_splits, 1):
        ws = torch.full((c * M * N,), NAN, dtype=torch.float32, device=DEV)
        obuf, o = _nan_out(M, I)
        SkinnyGemm(xd, stacked, None, None, ws, max_splits=c, silu_out=o).run()
        torch.cuda.synchronize()
        n = KT.k_slices_written(ws, M, N, c)
        assert n == expected_splits(M, N, K, c), (c, n)
        _canary_ok(obuf, M, I)
        part = ws[:n * M * N].view(n, M, N).cpu()
        acc = part[0].clone()
        for s in range(1, n):
            acc += part[s]
        outs[c], sums[c] = o, acc
    o3buf, o3 = _nan_out(M, I)
    SkinnyGemm(xd, interleave_gate_rows(w1.to(DEV), w2.to(DEV)), None, None, None, silu_out=o3, interleaved=True).run()
    torch.cuda.synchronize()
    _canary_ok(o3buf, M, I)
    ref_a, s_a = KT.gemm_ref(x, w1)
    ref_b, s_b = KT.gemm_ref(x, w2)
    for c, acc in sums.items():
        for half, ref, S in ((acc[:, :I], ref_a, s_a), (acc[:, I:], ref_b, s_b)):
            err = (half.to(F64) - ref).abs()
            assert bool((err <= KT.GEMM_C * S).all()), (c, float((err / S).max()))
        KT._check_gating(f"wide fin_mode 2 M {M} K {K} I {I} splits {expected_splits(M, N, K, c)}", outs[c], acc[:, :I], acc[:, I:])
    assert torch.equal(o3, outs[1]), "in-epilogue gating (fin_mode 3) != finalize gating (fin_mode 2) with one K slice"
    ref, _ = KT._gating_chain(ref_a, ref_b)
    eq = float((o3.cpu().to(F64) == ref).to(F64).mean())
    print(f"[wide] fin_mode 3 M {M} K {K} I {I}: bit-equal to the chain of the float64 sums {eq:.5f}")
    assert eq >= 0.98


# -------------------------------------------------------------------------------------- the same rows at two widths
@pytest.mark.parametrize("N,K,max_splits", [(1024, 4288, 1), (3072, 1024, 1), (512, 4160, 4)])
def test_same_rows_at_m128_and_as_half_of_m256(N, K, max_splits):
    """128 X rows through an M = 128 plan (wgmma N 128) and as the first and the second half of an M = 256 plan (N 256),
    with the same split count: every output within the bound, and the two widths agree bit for bit."""
    g = torch.Generator().manual_seed(N + K)
    x = KT._randn(g, 128, K)
    other = KT._randn(g, 128, K, scale=3.0)
    w = KT._randn(g, N, K, scale=K ** -0.5).to(DEV)
    ref, S = KT.gemm_ref(x, w.cpu())

    def run(X):
        M = X.shape[0]
        ws = torch.full((max_splits * M * N,), NAN, dtype=torch.float32, device=DEV)
        o = torch.full((M, N), NAN, dtype=BF, device=DEV)
        SkinnyGemm(X.to(DEV).contiguous(), w, o, None, ws, max_splits=max_splits).run()
        torch.cuda.synchronize()
        return o, max(1, KT.k_slices_written(ws, M, N, max_splits))

    o128, n128 = run(x)
    lo, n_lo = run(torch.cat([x, other]))
    hi, n_hi = run(torch.cat([other, x]))
    assert n128 == n_lo == n_hi == expected_splits(128, N, K, max_splits) == expected_splits(256, N, K, max_splits)
    for name, o in (("M 128", o128), ("M 256 rows 0..127", lo[:128]), ("M 256 rows 128..255", hi[128:])):
        KT.check_bound(f"two widths N {N} K {K} {name}", o, ref, KT.GEMM_C * S, 0.99)
    for name, o in (("rows 0..127", lo[:128]), ("rows 128..255", hi[128:])):
        eq = float((o == o128).float().mean())
        print(f"[wide] N {N} K {K} splits {n128}: M 256 {name} bit-equal to M 128 for {eq:.6f} of the outputs")
        # each output sums the same 16-element products in the same K order at either wgmma width
        assert torch.equal(o, o128), f"M 256 {name} differs from M 128"


def test_m257_is_rejected():
    x = torch.zeros(257, 64, dtype=BF, device=DEV)
    w = torch.zeros(128, 64, dtype=BF, device=DEV)
    out = torch.zeros(257, 128, dtype=BF, device=DEV)
    with pytest.raises(RstnetError, match="M<=256"):
        SkinnyGemm(x, w, out, None, None)
    assert MAX_STREAMS == 256


# ------------------------------------------------------------------------------------------------- whole LM, B = 256
def _config(cfg):
    return Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                  n_query_groups=cfg.n_kv, rotary_percentage=cfg.rotary_percentage, rope_adjustments=cfg.rope_adjustments,
                  intermediate_size=cfg.intermediate_size, norm_eps=cfg.norm_eps, padded_vocab_size=cfg.padded_vocab_size,
                  audio_card=cfg.audio_card, n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim,
                  codecformer_heads=cfg.codecformer_heads, codecformer_layers=cfg.codecformer_layers,
                  codecformer_dim_feedforward=cfg.codecformer_dim_feedforward, context=cfg.context)


def _build(cfg, seed):
    w32 = L.synthetic_weights(cfg, seed=seed, dtype=torch.float32, std=0.05)
    m = GPT(_config(cfg))
    m.load_state_dict(w32, strict=True)
    return m.to(DEV, BF).eval(), {k: v.to(DEV, BF) for k, v in w32.items()}


@pytest.fixture(scope="module")
def small256():
    m, w = _build(L.SMALL, 7)
    return m, w, L.SMALL


@pytest.fixture(scope="module")
def gqa256():
    cfg = dataclasses.replace(L.SMALL, n_query_groups=2, rotary_percentage=0.5,
                              rope_adjustments={"factor": 8.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                                "original_max_seq_len": 32})
    m, w = _build(cfg, 17)
    return m, w, cfg


def _cos(a, b):
    a, b = a.float().flatten().cpu(), b.float().flatten().cpu()
    return float(torch.dot(a, b) / (a.norm() * b.norm()).clamp(min=1e-12))


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-6))


def _seqs(B, n, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        s = torch.randint(0, 2048, (B, 9, 1), generator=g)
        s[:, 0] = torch.randint(0, 128256, (B, 1), generator=g)
        out.append(s.to(DEV))
    return out


def _vs_oracle(m, w, cfg, B, steps, seed):
    """`steps` teacher-forced frames (the ring wraps at context 16) against the oracle on the same GPU in bf16:
    transformer_out, text logits and the 8 depth logits of every row; greedy decisions counted against the oracle's."""
    gs = L.GPTStream(w, cfg, B)
    m.use_cuda_graphs = True
    agree = total = 0
    with m.streaming(B):
        for step, seq in enumerate(_seqs(B, steps, seed)):
            with torch.no_grad():
                r_out, r_tl = gs.forward_global(seq)
            out, tl = m.forward_global(seq)
            assert _cos(out, r_out) >= 0.999 and _rel(out, r_out) <= 5e-2, (step, _cos(out, r_out), _rel(out, r_out))
            assert _cos(tl, r_tl) >= 0.999 and _rel(tl, r_tl) <= 5e-2, (step, _cos(tl, r_tl), _rel(tl, r_tl))
            toks = r_tl.float().argmax(-1)
            agree += int((tl.float().argmax(-1) == toks).sum()); total += B
            gs.start_depth()
            with m.codecformer.streaming(B):
                prev = toks[:, :, None]
                for k in range(cfg.dep_q):
                    with torch.no_grad():
                        r_lg = gs.forward_codecformer(k, prev, r_out)
                    lg = m.forward_codecformer(k, prev, r_out)
                    assert _cos(lg, r_lg) >= 0.999 and _rel(lg, r_lg) <= 5e-2, (step, k, _cos(lg, r_lg), _rel(lg, r_lg))
                    prev = r_lg.float().argmax(-1)
                    agree += int((lg.float().argmax(-1) == prev).sum()); total += B
    print(f"[wide] B {B}: greedy decisions equal to the oracle's {agree}/{total}")
    assert agree >= 0.9 * total


def test_lm_b256_forward_global_vs_oracle(small256):
    m, w, cfg = small256
    _vs_oracle(m, w, cfg, 256, 18, 1)


def test_lm_b256_forward_step_greedy_sampled_and_graphs(small256):
    """forward_step at B = 256: greedy tokens == the stepwise API's argmaxes, a CUDA-graph replay == eager, and sampled
    audio ids stay below audio_valid."""
    m, w, cfg = small256
    B = 256
    seqs = _seqs(B, 4, 3)
    runs = {}
    for graphs in (True, False):
        m.use_cuda_graphs = graphs
        with m.streaming(B):
            runs[graphs] = [m.forward_step(s, use_sampling=False) for s in seqs]
    for a, b in zip(runs[True], runs[False]):
        assert torch.equal(a, b), "CUDA-graph replay differs from eager"
    m.use_cuda_graphs = True
    stepwise = []
    with m.streaming(B):
        for s in seqs:
            out, tl = m.forward_global(s)
            toks = [tl.float().argmax(-1)[:, 0]]
            with m.codecformer.streaming(B):
                prev = toks[0].view(B, 1, 1)
                for k in range(cfg.dep_q):
                    prev = m.forward_codecformer(k, prev, out).float().argmax(-1)
                    toks.append(prev[:, 0, 0])
            stepwise.append(torch.stack(toks, 1))
    for a, b in zip(runs[True], stepwise):
        assert torch.equal(a, b)
    with m.streaming(B):
        t = m.forward_step(seqs[0], use_sampling=True)
        assert t.shape == (B, 9) and int(t[:, 1:].max()) < 2049 and int(t.min()) >= 0
        for s in seqs[1:]:
            t = m.forward_step(s, use_sampling=True, top_k=30, temp=0.8, audio_valid=2048)
            assert int(t[:, 1:].max()) < 2048 and int(t.min()) >= 0


def test_lm_b256_reset_one_stream_and_hold_one(small256):
    """reset_streaming(streams=[200]) makes row 200 reproduce a fresh stream bit for bit while the other rows continue;
    a row held for two frames (set_active_streams) continues afterwards exactly as if those frames never happened."""
    m, w, cfg = small256
    B, r, h = 256, 200, 77
    seqs = _seqs(B, 10, 21)
    m.use_cuda_graphs = True
    with m.streaming(B):
        base = [m.forward_step(s, use_sampling=False) for s in seqs]
    with m.streaming(B):
        for t in range(4):
            m.forward_step(seqs[t], use_sampling=False)
        m.reset_streaming(streams=[r])
        got = []
        for t in range(4, 10):
            s = seqs[t].clone()
            s[r] = seqs[t - 4][r]
            got.append(m.forward_step(s, use_sampling=False))
    others = torch.arange(B) != r
    for i, t in enumerate(range(4, 10)):
        assert torch.equal(got[i][others.to(DEV)], base[t][others.to(DEV)]), "other rows must be undisturbed"
        assert torch.equal(got[i][r], base[t - 4][r]), "the reset row must reproduce a fresh stream"
    mask = torch.ones(B, dtype=torch.int64)
    mask[h] = 0
    with m.streaming(B):
        held = []
        for t in range(10):
            if t in (3, 4):
                m.set_active_streams(mask)
                s = seqs[t].clone()
                s[h] = seqs[(t + 5) % 10][h]                      # what a held row is fed must not matter
            else:
                m.set_active_streams(None)
                s = seqs[t].clone()
                if t > 4:
                    s[h] = seqs[t - 2][h]
            held.append(m.forward_step(s, use_sampling=False))
        assert int(m._state.offset[h]) == 8 and int(m._state.offset[0]) == 10
    for t in range(10):
        if t not in (3, 4):
            assert torch.equal(held[t][h], base[t if t < 3 else t - 2][h]), t
        keep = (torch.arange(B) != h).to(DEV)
        assert torch.equal(held[t][keep], base[t][keep]), t


def test_gqa_b256_wrapped_ring_vs_oracle(gqa256):
    """GQA (2 KV groups), rotary_percentage 0.5 and Llama-3.1 rope adjustments at B = 256 over a wrapped ring."""
    m, w, cfg = gqa256
    _vs_oracle(m, w, cfg, 256, 20, 2)


def test_gqa_prefill_b200_equals_single_steps(gqa256):
    """forward_global over 10 positions at B = 200 (one position per pass above 128 streams) leaves the rings and outputs
    that 10 single steps leave, bit for bit."""
    m, w, cfg = gqa256
    B, T = 200, 10
    seqs = _seqs(B, T + 1, 4)
    full = torch.cat(seqs[:T], dim=2)
    m.use_cuda_graphs = False
    with m.streaming(B):
        o_chunk, l_chunk = m.forward_global(full)
        kv_chunk = [k.clone() for k in m._state.kv]
        assert int(m._state.offset[0]) == T
        nxt_a = m.forward_global(seqs[T])[0]
    with m.streaming(B):
        outs, lgs = zip(*[m.forward_global(seqs[f]) for f in range(T)])
        kv_step = [k.clone() for k in m._state.kv]
        nxt_b = m.forward_global(seqs[T])[0]
    for a, b in zip(kv_chunk, kv_step):
        assert torch.equal(a, b)
    assert torch.equal(o_chunk, torch.cat(outs, 1)) and torch.equal(l_chunk, torch.cat(lgs, 1)) and torch.equal(nxt_a, nxt_b)
    with m.streaming(B):
        m.prefill(full)
        for a, b in zip(m._state.kv, kv_step):
            assert torch.equal(a, b)


def test_streaming_scope_limit(small256):
    m, w, cfg = small256
    with pytest.raises(RstnetError, match="256"):
        m.streaming_forever(257)
    m._state = None


# ----------------------------------------------------------------------------------------------------- Moshi twin
def test_moshi_lmgen_b256_vs_oracle():
    """LMGen.step at B = 256 on the small Moshi config: every (text, audio) decision of the greedy closed loop under the
    oracle teacher-forced with those tokens, as test_moshi_gpu.test_lmgen_step_closed_loop checks at B = 2."""
    from rstnet_b200.moshi import LMGen, LMModel
    cfg, B = MO.SMALL, 256
    w = MO.synthetic_weights(cfg, seed=5)
    m = LMModel(**cfg.reference_kwargs())
    m.load_state_dict(w, strict=True)
    m = m.to(DEV, BF).eval()
    g = torch.Generator().manual_seed(9)
    inputs = torch.randint(0, cfg.card, (5, B, cfg.n_q - cfg.dep_q, 1), generator=g)
    gen = LMGen(m, use_sampling=False)
    ora = MO.LMGenOracle({k: v.to(BF) for k, v in w.items()}, cfg, B)
    exact = n = 0
    worst = 0.0
    with gen.streaming(B), torch.no_grad():
        for t in range(inputs.shape[0]):
            o = gen.step(inputs[t].to(DEV))
            assert (o is None) == (t < max(cfg.delays))
            pos = gen._st.offset % gen._st.cache.shape[2]
            ours = gen._st.cache[:, :cfg.dep_q + 1, pos].cpu()
            ora.step(inputs[t], force=ours)
            _, _, text_logits, alog = ora.last
            lt = text_logits.float()[:, 0, 0]
            d = [lt.max(-1).values - lt.gather(1, ours[:, :1])[:, 0]]
            la = alog.float()
            d.append((la.max(-1).values - la.gather(2, ours[:, 1:, None])[:, :, 0]).flatten())
            d = torch.cat(d)
            worst = max(worst, float(d.max()))
            exact += int((d == 0).sum()); n += d.numel()
    print(f"[wide] moshi LMGen B {B}: {exact}/{n} decisions are the oracle's exact argmax; worst deficit {worst:.3f}")
    assert worst <= 0.1 and exact >= 0.8 * n


# ------------------------------------------------------------------------------------------------------- serving
def test_duplex_engine_capacity_256():
    """DuplexEngine + FrameScheduler with 256 rows (250 sessions, a tiny LM) for four ticks, some sessions silent on some
    ticks: every session that pushed a frame gets exactly that tick's output; 257 rows are refused."""
    from specs import mimi_spec as S
    from rstnet_b200.codec import MimiCodec
    from rstnet_b200.serve import DuplexEngine, FrameScheduler
    codec = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    codec.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
    codec = codec.to(DEV).eval()
    lm, _ = _build(L.SMALL, 7)
    with pytest.raises(RstnetError, match="256"):
        DuplexEngine(codec, lm, 257)
    audio = S.synthetic_audio(4, 1920 * 4, seed=55)
    eng = DuplexEngine(codec, lm, 256)
    sch = FrameScheduler(eng, 256)
    sessions = list(range(250))
    for s in sessions:
        sch.admit(s)
    counts = dict.fromkeys(sessions, 0)
    for tick in range(4):
        pushed = [s for s in sessions if (s + tick) % 7 != 0]        # the others are held this tick
        for s in pushed:
            sch.push(s, audio[s % 4, 0, tick * 1920:(tick + 1) * 1920])
        out = sch.tick()
        assert sorted(out) == pushed
        for s, (tok, pcm) in out.items():
            assert tok.shape == (9,) and pcm.shape == (1920,) and bool(torch.isfinite(pcm).all())
            assert int(tok[1:].max()) < 2048 and int(tok.min()) >= 0
            counts[s] += 1
    assert all(counts[s] == sum((s + t) % 7 != 0 for t in range(4)) for s in sessions)
    assert len(eng.latencies_ms) == 4 and sch.free_rows() == 6
