"""Checks of the sampler's host restatement (tests/sampler_restatement.py) on the CPU: its nucleus kept sets against the
float64 oracle and the reference's kept sets, its top-k sets against a sort, its noise against softmax frequencies (the
only statistical check), and its score bounds against adversarial fp32 evaluations of the kernel's expressions."""
import os

import numpy as np
import pytest
import torch

import sampler_restatement as S
from oracle import sampling_oracle as O
from oracle.gen_golden_sampling import row_logits
from rvq_restatement import fma32

MARGIN = 3e-5   # as tests/test_sampling_params_cpu.py: the reference's fp32 cumsum against float64


def _fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "sampling_top_p.npz"))
    for j in range(len(g["seed"])):
        r = (int(g["seed"][j]), int(g["V"][j]), int(g["n_valid"][j]), str(g["kind"][j]), float(g["scale"][j]),
             float(g["temp"][j]), float(g["p"][j]))
        yield r, np.unpackbits(g["kept_bits"][j])[:r[2]].astype(bool), row_logits(*r)


def test_hash_and_uniform():
    """uint32 wraparound, and the fp32 uniform: exact below 2^23, rounded to even above, 1 at the very top"""
    h = S.hash_u32(2 ** 32 - 1, 2 ** 32 + 5, -1, np.arange(4))
    assert h.dtype == np.uint32
    assert np.array_equal(h, S.hash_u32(2 ** 32 - 1, 5, 2 ** 32 - 1, np.arange(4)))
    u = np.array([0, 255, 256, (2 ** 23 - 1) << 8, (2 ** 23 + 1) << 8, 0xFFFFFFFF], dtype=np.uint32)
    uni = S.uniform32(u)
    assert uni.dtype == np.float32
    assert uni[0] == uni[1] == np.float32(0.5 * 2.0 ** -24) and uni[2] == np.float32(1.5 * 2.0 ** -24)
    assert uni[3] == np.float32((2 ** 23 - 0.5) * 2.0 ** -24)
    assert uni[4] == np.float32((2 ** 23 + 2) * 2.0 ** -24)      # 2^23 + 1.5 rounds to even
    assert uni[5] == 1.0 and S.gumbel(uni[5:]) == np.inf


def test_parameter_resolution():
    R = S.resolve
    assert R(100, 0, 5, 1.0, 0.0) == S.RowParams(100, "topk", 5, np.float32(1.0), np.float32(0.0))
    assert R(100, 200, 500, 1.0, 0.0).top_k == 100 and R(100, 7, 500, 1.0, 0.0).top_k == 7
    assert R(100, 7, 500, 1.0, 0.0, nv_row=-3).n_valid == 100 and R(100, 7, 500, 1.0, 0.0, nv_row=-3).top_k == 100
    assert R(5000, 0, 0, 1.0, 0.0, table=(3000, 0.7, 0.0)).top_k == 1024
    assert R(5000, 0, 0, 1.0, 0.0, nv_row=9, table=(3000, 0.7, 0.0)).top_k == 9
    for t in (0.0, -1.0, float("nan")):
        assert R(50, 0, 0, 1.0, 0.0, table=(-1, t, 0.5)).mode == "argmax"
    assert R(50, 0, 0, 1.0, 0.0, table=(-1, 0.7, float("nan"))).mode == "multinomial"
    assert R(50, 0, 0, 1.0, 0.0, table=(5, 0.7, 0.9)).mode == "nucleus"
    assert R(50, 0, 5, 0.7, 1.0).mode == "topk" and R(50, 0, 0, 0.7, 0.5).mode == "argmax"


def test_nucleus_kept_sets_equal_the_oracle_and_the_reference(golden_dir):
    """the 2^-40 fixed-point cut against the float64 masses (the same prefix of the order up to ranks whose mass before
    lies within 1e-6 of p: the weights' truncation) and against the reference's kept sets (within MARGIN, as the
    float64 oracle itself); the narrow and wide sets differ only there"""
    n = 0
    for (seed, V, n_valid, kind, scale, temp, p), ref, lg in _fixture(golden_dir):
        x = S._values(lg, n_valid)
        mine = np.zeros(n_valid, dtype=bool)
        mine[S.nucleus_exact(x, np.float32(temp), np.float32(p))] = True
        order, before, _ = O.nucleus(lg, n_valid, temp)
        n_mine, n_ora, n_ref = int(mine.sum()), int(O.kept_set(lg, n_valid, temp, p).sum()), int(ref.sum())
        assert np.array_equal(mine[order[:n_mine]], np.ones(n_mine, dtype=bool)), kind   # a prefix of the same order
        lo, hi = sorted((n_mine, n_ora))
        assert np.all(np.abs(before[lo:hi] - p) <= 1e-6), (seed, kind, n_mine, n_ora)
        lo, hi = sorted((n_mine, n_ref))
        assert np.all(np.abs(before[lo:hi] - p) <= MARGIN), (seed, kind, n_mine, n_ref)
        ids, n_narrow, n_wide = S.nucleus_sets(x, np.float32(temp), np.float32(p))
        assert n_narrow <= n_mine <= n_wide
        assert np.all(np.abs(before[n_narrow:n_wide] - p) <= 1e-5), (seed, kind, n_narrow, n_wide)
        n += 1
    assert n == 39


@pytest.mark.parametrize("V,k", [(8, 3), (2050, 64), (4097, 65), (32000, 1024)])
def test_topk_sets_equal_a_sort(V, k):
    g = torch.Generator().manual_seed(V)
    bits = torch.cat([torch.arange(0x0001, 0x7F80), torch.arange(0x8001, 0xFF80)])   # every finite bf16 but -0, once
    for _ in range(4):
        pick = bits[torch.randperm(len(bits), generator=g)[:V]]
        x = pick.to(torch.int16).view(torch.bfloat16).float().numpy()
        assert len(np.unique(x)) == V
        want = torch.topk(torch.from_numpy(x), k).indices.numpy()
        assert set(S.topk_set(x, k).tolist()) == set(want.tolist())
        assert np.array_equal(S.topk_set(x, k), want)                          # also in order


def test_order_ties_signed_zeros_and_nan():
    x = np.array([0.0, -0.0, np.nan, 1.0, -0.0, 0.0, -np.inf, np.nan, 1.0], dtype=np.float32)
    assert S.order(x).tolist() == [3, 8, 0, 1, 4, 5, 6]
    assert S.topk_set(x, 4).tolist() == [3, 8, 0, 1]


def test_draws_match_softmax_frequencies():
    """Over 40 000 noise keys: the Gumbel-max draw of l / temp + G (multinomial) and the rank-keyed race w_r / e_r
    (top_k <= 64) both follow softmax(l / temp) within 1e-2."""
    V, temp, n = 12, np.float32(0.8), 40000
    x = torch.linspace(-1.5, 1.0, V).to(torch.bfloat16).float().numpy()
    p = np.exp(x / float(temp) - np.max(x / float(temp)))
    p /= p.sum()
    keys = np.arange(n)[:, None]
    inv_t = np.float32(1.0) / temp
    G = S.gumbel(S.uniform32(S.hash_u32(7, 3, keys, np.arange(V)[None, :])))
    freq = np.bincount(np.argmax(x * float(inv_t) + G, axis=1), minlength=V) / n
    assert np.abs(freq - p).max() < 1e-2, np.abs(freq - p).max()
    order = S.order(x)
    v = x[order]
    w = np.exp((v - v[0]) / float(temp))
    e = -np.log(S.uniform32(S.hash_u32(7, 3, keys, np.arange(V)[None, :])).astype(np.float64))
    freq = np.bincount(order[np.argmax(w / e, axis=1)], minlength=V) / n
    assert np.abs(freq - p).max() < 1e-2, np.abs(freq - p).max()
    # and draw() agrees with the vectorised race on every key
    prm = S.resolve(V, 0, -1, float(temp), 0.0)
    got = [S.draw(torch.from_numpy(x).to(torch.bfloat16), prm, 7, 3, k) for k in range(300)]
    assert all(d.ok == {int(np.argmax(x * float(inv_t) + G[k]))} for k, d in enumerate(got))


def _ulps(v32: np.ndarray, n: int) -> np.ndarray:
    """v32 moved n fp32 ulps (n > 0 up, < 0 down)"""
    out = v32.copy()
    for _ in range(abs(n)):
        out = np.nextafter(out, np.float32(np.inf if n > 0 else -np.inf)).astype(np.float32)
    return out


def test_score_bounds_cover_fp32_evaluations():
    """Every fp32 evaluation the kernel may make, with logf and expf at the ends of their documented error (1 and 2 ulp
    from the correctly rounded value) and l * inv_t + g with and without FFMA contraction, lies inside the bounds."""
    g = torch.Generator().manual_seed(3)
    l = (torch.randn(20000, generator=g) * torch.tensor([0.01, 1.0, 30.0, 3e3]).repeat(5000)).to(torch.bfloat16).float().numpy()
    ids = np.arange(len(l))
    for temp in (np.float32(0.3), np.float32(0.7), np.float32(1.5)):
        inv_t = np.float32(1.0) / temp
        lo, hi = S.multinomial_scores(l, ids, inv_t, 5, 9, 11)
        uni = S.uniform32(S.hash_u32(5, 9, 11, ids))
        a0 = np.log(uni.astype(np.float64)).astype(np.float32)
        for da in (-1, 1):
            a = _ulps(a0, da)
            c0 = np.log(-a.astype(np.float64)).astype(np.float32)
            for dc in (-1, 1):
                gk = -_ulps(c0, dc)
                fused = fma32(torch.from_numpy(l), torch.tensor(inv_t), torch.from_numpy(gk)).numpy()
                plain = (l * inv_t) + gk
                for s in (fused, plain):
                    assert np.all((lo <= s) & (s <= hi)), temp
        # top_k <= 64: w / e with expf and logf at their error ends
        v = np.sort(l[:64])[::-1].copy()
        lo, hi = S.rank_scores(v, temp, 5, 9, 11)
        q = (v - v[0]) / temp
        e0 = (-np.log(S.uniform32(S.hash_u32(5, 9, 11, np.arange(64))).astype(np.float64))).astype(np.float32)
        w0 = np.exp(q.astype(np.float64)).astype(np.float32)
        for dw in (-2, 2):
            for de in (-1, 1):
                s = np.maximum(_ulps(w0, dw), np.float32(0)) / _ulps(e0, de)   # expf is never negative
                assert np.all((lo <= s) & (s <= hi)), temp


def test_edge_rows():
    """rows with no candidate above -inf draw 0 in every mode; a +inf logit wins the score-based modes; NaN is never
    drawn; overflow of l / temp to +-inf"""
    bf = torch.bfloat16
    modes = [(0, 1.0, 0.0), (1, 0.7, 0.0), (5, 0.7, 0.0), (300, 0.7, 0.0), (-1, 0.7, 0.0), (-1, 0.7, 0.9), (5, 0.7, 0.5)]
    rows = {"ninf": torch.full((50,), -np.inf), "nan": torch.full((50,), np.nan),
            "mix": torch.tensor([np.nan, -np.inf] * 25)}
    for name, row in rows.items():
        for tk, te, tp in modes:
            assert S.draw(row.to(bf), S.resolve(50, 0, tk, te, tp), 1, 2, 3).ok == {0}, (name, tk, tp)
    inf = torch.randn(50, generator=torch.Generator().manual_seed(1))
    inf[[17, 30]] = np.nan
    inf[23] = np.inf
    for tk, te, tp in modes:
        d = S.draw(inf.to(bf), S.resolve(50, 0, tk, te, tp), 1, 2, 3)
        assert d.ok == {23}, (tk, tp, d)
    big = torch.tensor([3e38, -3e38, 1.0, -3e38]).to(bf)
    for tk, te, tp in modes:
        assert S.draw(big, S.resolve(4, 0, tk, 0.3, tp), 1, 2, 3).ok == {0}, (tk, tp)
    neg = torch.tensor([-3e38] * 4).to(bf)
    assert S.draw(neg, S.resolve(4, 0, -1, 0.3, 0.0), 1, 2, 3).ok == {0}       # every score overflows to -inf
