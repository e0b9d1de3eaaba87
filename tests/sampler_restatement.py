"""Host restatement of the LM sampler (rstnet_lm_sample_params_bf16, sample_row / sample_kernel in
rstnet_b200/csrc/lm_small.cu): every draw as a function of the launch inputs.

The noise is a counter-based hash, hash_u32(seed, step, key, id or rank), whose top 24 bits give the uniform
(float(u >> 8) + 0.5f) * 2^-24 in fp32 (restated here in fp32: from 2^23 on, + 0.5f rounds to even, so u >> 8 =
2^24 - 1 gives exactly 1 and a Gumbel noise of +inf).  The kept sets are integer and order decisions on bf16 values,
restated exactly.  The scores are evaluated in float64 with a bound on the kernel's fp32 evaluation (the library is built
without fast math: logf within 1 ulp, expf within 2, divisions and the rest correctly rounded; `l * inv_t + g` with or
without FFMA contraction).  So the answer is the set of ids the kernel may draw: one id, or a few near-ties whose scores
lie within the bound of the best.

Modes, as the kernel resolves them:
* argmax (top_k == 0): the first maximum;
* top-k (1..1024): the first top_k ids in the order (value desc, index asc) under float comparison, NaN excluded.  Up to
  64 the draw is the first maximum over ranks r of w_r / e_r, w_r = expf((v_r - v_0) / temp) (1 for +inf), e_r =
  -logf(uni(rank r)); above 64 the first maximum (lowest id on equal scores) of the multinomial score l * inv_t + Gumbel
  over the kept ids, the noise keyed by id;
* multinomial (top_k < 0): the same score over every id < n_valid;
* nucleus (top_k != 0, 0 < top_p < 1): the ids whose 2^-40 fixed-point mass before them in the order is <=
  floor((double)top_p * Z), then the multinomial score over them.  The weights floor(expf(x) * 2^40) are known within
  expf's 2 ulp, so ids near the cut are ambiguous; every prefix between the narrow and the wide kept set is allowed.
* no kept id scoring above -inf (in particular no id above -inf): id 0.

The path constants (SAMPLE_CAND, the candidate list above 4096 ids, the threshold select above top_k 64) choose test
shapes only; nothing here depends on them except the table clamp of top_k to SAMPLE_CAND.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

SAMPLE_CAND = 1024
U32 = np.uint32
INF = np.inf
REL_G = 2.0 ** -21                 # -logf(-logf(u)): two logf of 1 ulp each, with a factor 2 to spare
REL_EXP = 2.0 ** -21               # expf: 2 ulp, with a factor 2 to spare
REL_LOG = 2.0 ** -22               # logf: 1 ulp, with a factor 2 to spare
TINY = 2.0 ** -148                 # absolute slack for results in fp32's subnormal range


def hash_u32(a, b, c, d) -> np.ndarray:
    """the kernel's hash_u32 with uint32 wraparound; arguments broadcast"""
    a, b, c, d = (np.asarray(np.asarray(t, dtype=np.int64) & 0xFFFFFFFF, dtype=U32) for t in (a, b, c, d))
    with np.errstate(over="ignore"):
        h = (a * U32(0x9E3779B1)) ^ ((b + U32(0x7F4A7C15)) * U32(0x85EBCA77)) ^ ((c + U32(0x165667B1)) * U32(0xC2B2AE3D)) \
            ^ (d * U32(0x27D4EB2F))
        h = h ^ (h >> U32(16))
        h = h * U32(0x7FEB352D)
        h = h ^ (h >> U32(15))
        h = h * U32(0x846CA68B)
        h = h ^ (h >> U32(16))
    return h


def uniform32(u: np.ndarray) -> np.ndarray:
    """((float)(u >> 8) + 0.5f) * (1.0f / 16777216.0f) in fp32: in (0, 1]"""
    return (np.asarray(u >> U32(8)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -24)


def gumbel(uni: np.ndarray) -> np.ndarray:
    """-log(-log(uni)) in float64 of the fp32 uniform (+inf at uni == 1)"""
    with np.errstate(divide="ignore"):
        return -np.log(-np.log(uni.astype(np.float64)))


# ------------------------------------------------------------------------------------------------ parameters
@dataclass(frozen=True)
class RowParams:
    n_valid: int
    mode: str          # "argmax" | "topk" | "multinomial" | "nucleus"
    top_k: int
    temp: np.float32
    top_p: np.float32


def resolve(V: int, n_valid: int, top_k: int, temp: float, top_p: float, nv_row=None, table=None) -> RowParams:
    """the entry point's and sample_kernel's parameter resolution for one row: n_valid (scalar, or the row's table entry
    nv_row) outside (0, V] is V; top_k is clamped to it; a settings table entry (top_k, temp, top_p) is also clamped to
    SAMPLE_CAND, temp <= 0 or NaN means argmax, and a top_p that is not >= 0 is 0"""
    if n_valid <= 0 or n_valid > V:
        n_valid = V
    if nv_row is None:
        top_k = min(top_k, n_valid)
    else:
        n_valid = int(nv_row)
        if n_valid <= 0 or n_valid > V:
            n_valid = V
        top_k = min(top_k, n_valid)
    temp, top_p = np.float32(temp), np.float32(top_p)
    if table is not None:
        top_k, temp, top_p = int(table[0]), np.float32(table[1]), np.float32(table[2])
        top_k = min(top_k, SAMPLE_CAND, n_valid)
        if not temp > 0:
            top_k, temp = 0, np.float32(1.0)
        if not top_p >= 0:
            top_p = np.float32(0.0)
    if top_k != 0 and 0 < top_p < 1:
        mode = "nucleus"
    elif top_k < 0:
        mode = "multinomial"
    elif top_k == 0:
        mode = "argmax"
    else:
        mode = "topk"
    return RowParams(n_valid, mode, int(top_k), temp, top_p)


# ------------------------------------------------------------------------------------------------ kept sets
def _values(row, n_valid: int) -> np.ndarray:
    """the first n_valid logits of a bf16 row as float32 (exact)"""
    return torch.as_tensor(row)[:n_valid].to(torch.bfloat16).float().numpy()


def order(x: np.ndarray) -> np.ndarray:
    """the non-NaN ids in the order (value desc, index asc) under float comparison (-0 == +0)"""
    ids = np.flatnonzero(~np.isnan(x))
    return ids[np.lexsort((ids, -x[ids]))]


def topk_set(x: np.ndarray, k: int) -> np.ndarray:
    return order(x)[:k]


def nucleus_weights(x: np.ndarray, temp: np.float32):
    """(W, dW): each id's 2^-40 fixed-point weight floor(expf((l - max) * inv_t) * 2^40) as the float64 expf of the
    kernel's exact fp32 argument, and the bound on its distance to the kernel's (int64 [n] each; NaN ids weigh 0)"""
    inv_t = np.float32(1.0) / temp
    mx = np.float32(np.max(x, initial=-INF, where=~np.isnan(x)))
    with np.errstate(invalid="ignore", over="ignore"):
        arg = (x - mx) * inv_t                        # fp32, as the kernel evaluates it
        w = np.exp(arg.astype(np.float64))
    w = np.where(np.isnan(w), 0.0, w)
    scaled = w * 2.0 ** 40
    W = np.floor(scaled).astype(np.int64)
    dW = np.where((w > 0) & (arg != 0), np.ceil(scaled * REL_EXP) + 1, 0).astype(np.int64)   # expf(0) is 1
    return W, dW


def nucleus_sets(x: np.ndarray, temp: np.float32, top_p: np.float32):
    """(ids in order, n_narrow, n_wide): the kept set is a prefix of the order holding at least n_narrow and at most
    n_wide ids; with exact weights it is the ids whose mass before them is <= floor((double)top_p * Z)"""
    ids = order(x)
    W, dW = nucleus_weights(x, temp)
    w, d = W[ids], dW[ids]
    before = np.concatenate([[0], np.cumsum(w)[:-1]])
    dbefore = np.concatenate([[0], np.cumsum(d)[:-1]])
    Z, D = int(w.sum()), int(d.sum())
    p = float(top_p)
    if D == 0:      # exact weights: the kernel's cut
        lo = hi = int(p * float(Z))
    else:
        lo, hi = int(p * float(max(Z - D, 0))) - 1, int(p * float(Z + D)) + 1
    n_narrow = max(int(np.sum(before + dbefore <= lo)), 1)
    maybe = np.flatnonzero(before - dbefore <= hi)     # (not monotone: ids of weight 0 carry a bound of 1 or 2)
    n_wide = max(int(maybe[-1]) + 1 if len(maybe) else 1, n_narrow)
    return ids, n_narrow, n_wide


def nucleus_exact(x: np.ndarray, temp: np.float32, top_p: np.float32) -> np.ndarray:
    """the kept ids with the nominal weights (no expf error): for the checks against the float64 oracle"""
    ids = order(x)
    W, _ = nucleus_weights(x, temp)
    w = W[ids]
    before = np.concatenate([[0], np.cumsum(w)[:-1]])
    cut = int(float(top_p) * float(int(w.sum())))
    keep = before <= cut
    keep[:1] = True
    return ids[keep]


# ------------------------------------------------------------------------------------------------ scores
def _rn32_bounds(t_lo: np.ndarray, t_hi: np.ndarray):
    """fp32 round-to-nearest of every real in [t_lo, t_hi] (float64 ends, each within one float64 rounding of the real
    end) lies in the returned fp32 values (as float64): the ends moved out by more than that rounding, then rounded"""
    with np.errstate(invalid="ignore", over="ignore"):
        lo = t_lo - np.where(np.isfinite(t_lo), np.abs(t_lo) * 2.0 ** -50, 0.0)
        hi = t_hi + np.where(np.isfinite(t_hi), np.abs(t_hi) * 2.0 ** -50, 0.0)
        return lo.astype(np.float32).astype(np.float64), hi.astype(np.float32).astype(np.float64)


def multinomial_scores(x: np.ndarray, ids: np.ndarray, inv_t: np.float32, seed: int, stepc: int, key: int):
    """(lo, hi): the kernel's fp32 score l * inv_t + (-logf(-logf(uni))) of each id lies in [lo, hi], fused (one
    rounding of l * inv_t + g) or not (l * inv_t rounded first); NaN: the score is NaN (never drawn); lo = -inf, hi = +inf:
    NaN or +inf (l * inv_t overflows to -inf in one form only, with a Gumbel noise of +inf)"""
    G = gumbel(uniform32(hash_u32(seed, stepc, key, ids)))
    eg = np.where(np.isinf(G), 0.0, REL_G * (1.0 + np.abs(G)))
    with np.errstate(invalid="ignore", over="ignore"):
        xs = x[ids].astype(np.float64) * float(inv_t)      # exact: bf16 x fp32
        xr = xs.astype(np.float32).astype(np.float64)      # rounded to fp32 first (inf on overflow)
        fl, fh = _rn32_bounds(xs + (G - eg), xs + (G + eg))
        ul, uh = _rn32_bounds(xr + (G - eg), xr + (G + eg))
    lo, hi = np.fmin(fl, ul), np.fmax(fh, uh)
    one_nan = np.isnan(fl) != np.isnan(ul)
    lo, hi = np.where(one_nan, -INF, lo), np.where(one_nan, INF, hi)
    both_nan = np.isnan(fl) & np.isnan(ul)
    return np.where(both_nan, np.nan, lo), np.where(both_nan, np.nan, hi)


def rank_scores(v: np.ndarray, temp: np.float32, seed: int, stepc: int, key: int):
    """(lo, hi) bounds on the top_k <= 64 scores w_r / e_r of the ranks r of values v (v[0] the largest); NaN: never"""
    r = np.arange(len(v))
    uni = uniform32(hash_u32(seed, stepc, key, r))
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        q = (v - v[0]) / temp                         # fp32 subtraction and true division, as the kernel
        w = np.exp(q.astype(np.float64))
        w = np.where(v == np.float32(INF), 1.0, w)
        wlo = np.maximum(w * (1 - REL_EXP) - TINY, 0.0)
        whi = np.where(w > 0, w * (1 + REL_EXP) + TINY, np.where(q == -INF, 0.0, TINY))
        whi = np.where(v == np.float32(INF), 1.0 + REL_EXP, whi)
        e = -np.log(uni.astype(np.float64))
        lo = np.maximum(wlo / (e * (1 + REL_LOG)) * (1 - 2.0 ** -23) - TINY, 0.0)
        hi = np.where(whi > 0, whi / (e * (1 - REL_LOG)) * (1 + 2.0 ** -23) + TINY, 0.0)
    never = uni == 1                                   # e = -0: the score is -inf or NaN
    return np.where(never, np.nan, lo), np.where(never, np.nan, hi)


def possible_winners(lo: np.ndarray, hi: np.ndarray) -> np.ndarray:
    """positions (in tie order: earlier wins equal scores) that may hold the first maximum of scores known to lie in
    [lo, hi]; scores never above -inf and NaN scores are never drawn"""
    ok = ~np.isnan(lo) & (hi > -INF)
    L = np.where(ok, lo, -INF)
    before = np.concatenate([[-INF], np.maximum.accumulate(L)[:-1]])
    after = np.concatenate([np.maximum.accumulate(L[::-1])[::-1][1:], [-INF]])
    return np.flatnonzero(ok & (hi > before) & (hi >= after))


def _winners_or(ids, lo, hi, fallback: int) -> set:
    """ids that may be drawn, plus the fallback when possibly no score is above -inf"""
    pos = possible_winners(lo, hi)
    out = {int(ids[p]) for p in pos}
    ok = ~np.isnan(lo) & (hi > -INF)
    if not ok.any() or np.max(np.where(ok, lo, -INF)) == -INF:
        out.add(fallback)
    return out


# ------------------------------------------------------------------------------------------------ draws
@dataclass
class Draw:
    ok: set            # the ids the kernel may draw
    mode: str
    kept: int          # size of the (narrow) kept set

    @property
    def exact(self) -> bool:
        return len(self.ok) == 1


def draw(row, prm: RowParams, seed: int, stepc: int, key: int) -> Draw:
    """the ids the kernel may draw for one row of logits (bf16, length >= prm.n_valid) with resolved parameters, noise
    keyed by (seed, stepc, key) (all taken as uint32)"""
    x = _values(row, prm.n_valid)
    seed, stepc, key = seed & 0xFFFFFFFF, stepc & 0xFFFFFFFF, key & 0xFFFFFFFF
    if not np.any(x > -INF):
        return Draw({0}, prm.mode, 0)
    inv_t = np.float32(1.0) / prm.temp
    if prm.mode == "argmax":
        return Draw({int(order(x)[0])}, "argmax", 1)
    if prm.mode == "multinomial":
        ids = np.flatnonzero(~np.isnan(x))
        lo, hi = multinomial_scores(x, ids, inv_t, seed, stepc, key)
        return Draw(_winners_or(ids, lo, hi, 0), "multinomial", len(ids))
    if prm.mode == "topk":
        kept = topk_set(x, prm.top_k)
        if prm.top_k <= 64:
            lo, hi = rank_scores(x[kept], prm.temp, seed, stepc, key)
            return Draw(_winners_or(kept, lo, hi, int(kept[0])), "topk", len(kept))
        ids = np.sort(kept)
        lo, hi = multinomial_scores(x, ids, inv_t, seed, stepc, key)
        return Draw(_winners_or(ids, lo, hi, 0), "topk", len(kept))
    ids, n_narrow, n_wide = nucleus_sets(x, prm.temp, prm.top_p)
    narrow = np.sort(ids[:n_narrow])
    lo, hi = multinomial_scores(x, narrow, inv_t, seed, stepc, key)
    ok = _winners_or(narrow, lo, hi, 0)
    if n_wide > n_narrow:
        # an ambiguous id may be kept, and then drawn if it may beat every surely kept id (a superset of the prefixes'
        # winners); each kept ambiguous id can only take the draw from the narrow set's winners, not add others
        amb = ids[n_narrow:n_wide]
        alo, ahi = multinomial_scores(x, amb, inv_t, seed, stepc, key)
        best = np.max(np.where(np.isnan(lo), -INF, lo), initial=-INF)
        ok |= {int(a) for a, h in zip(amb, ahi) if not np.isnan(h) and h >= best and h > -INF}
    return Draw(ok, "nucleus", n_narrow)


def draw_launch(logits: torch.Tensor, *, n_valid: int = 0, top_k: int = 0, temp: float = 1.0, top_p: float = 0.0,
                nv_rows=None, tables=None, seed: int = 0, step=None, step_rows=None, key_rows=None):
    """Draw per row of one rstnet_lm_sample_params_bf16 launch on logits [R, V] (bf16): the arguments as the entry point
    takes them; nv_rows [R] and tables (top_k [R], temp [R], top_p [R]) are the rows' table entries.  The noise key is
    (seed, step_rows[r], key_rows[r]) when step_rows is given, else (seed, step or 0, r)."""
    R, V = logits.shape
    lg = logits.detach().to("cpu")
    out = []
    for r in range(R):
        prm = resolve(V, n_valid, top_k, temp, top_p, None if nv_rows is None else nv_rows[r],
                      None if tables is None else (tables[0][r], tables[1][r], tables[2][r]))
        if step_rows is not None:
            stepc, key = int(step_rows[r]), int(key_rows[r])
        else:
            stepc, key = (0 if step is None else int(step)), r
        out.append(draw(lg[r], prm, seed, stepc, key))
    return out
