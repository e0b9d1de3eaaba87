"""Exact host restatement of the codec's RVQ encoder (rstnet_rvq_encode_f32, rstnet_b200/csrc/rvq.cu), plus the float64
nearest-centroid bound its choices must meet.

The kernel's arithmetic per (frame, level), on the fp32 residual r of dim components:

* acc_c = fmaf chain of (-2 r_k) * e_ck over k = 0 .. dim-1 in ascending order, starting at +0;
* xnorm = per lane s_lane = fmaf chain of h_d * h_d over d = lane, lane + 32, ... with h = -0.5f * (-2 r), then the xor
  butterfly 16, 8, 4, 2, 1 (fp32 addition is commutative, so each step is one plain fp32 add and every lane ends with
  the same value);
* d_c = sqrtf(fmaxf((acc_c + xnorm) + enorm_c, 0)), and the code is the first index of the minimum d;
* the next level's residual is r - e_prev[code] in fp32.

Every step is restated here with one correct rounding per fp32 operation, so the codes must equal the kernel's bit for
bit: no margins, no tolerated exceptions.  fmaf is the only operation float64 cannot evaluate in one rounding; `fma32`
restates it exactly (the product in float64, the sum rounded to odd at 53 bits, then to fp32).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

F32, F64 = torch.float32, torch.float64
U = 2.0 ** -24     # unit roundoff of fp32


def fma32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    """fmaf(a, b, c) on fp32 tensors, correctly rounded (round to nearest even), computed in float64.

    a * b of two fp32 values is exact in float64 (24 + 24 significant bits).  The sum with c is rounded to odd at 53
    bits: TwoSum gives the float64 sum s and its exact error; if the error is non-zero and s is even, s steps one
    float64 ulp toward the error.  Rounding a round-to-odd value of at least p + 2 bits to p bits is a correct rounding,
    so the final conversion to fp32 (24 bits, fewer in the subnormal range) is fmaf's result, ties and all.

    Only a float64 sum that lands exactly on an fp32 rounding boundary (a normal-range midpoint: the 29 bits below the
    fp32 ulp are 1000...0) or below 2^-126 can round differently from the exact sum, since any other boundary lying
    between the two would be a closer float64.  The TwoSum correction runs on those elements only; the result is the
    same as running it everywhere."""
    p = a.to(F64) * b.to(F64)
    c = c.to(F64)
    s = p + c
    bits = s.view(torch.int64)
    near = ((bits & _LOW29) == _HALF29) | (((bits >> 52) & 0x7FF) < 1023 - 126)
    if bool(near.any()):
        i = near.nonzero(as_tuple=True)
        pi, ci, si = p.expand_as(s)[i], c.expand_as(s)[i], s[i]
        bb = si - pi
        err = (pi - (si - bb)) + (ci - bb)
        fix = (err != 0) & ((si.view(torch.int64) & 1) == 0) & torch.isfinite(si)
        s[i] = torch.where(fix, torch.nextafter(si, torch.copysign(torch.full_like(si, math.inf), err)), si)
    return s.to(F32)


_LOW29, _HALF29 = (1 << 29) - 1, 1 << 28


def level_distances(r: torch.Tensor, E_l: torch.Tensor, en_l: torch.Tensor):
    """The kernel's fp32 (d2, d) of residuals r [n, dim] against centroids E_l [bins, dim] with norms en_l [bins]."""
    n, dim = r.shape
    r = r.to(F32)
    E_l = E_l.to(F32)
    m2 = -2.0 * r                                               # rs = -2 * residual (fp32, exact but restated)
    a64, e64 = m2.to(F64), E_l.t().to(F64).contiguous()        # fp32 values, held in float64 (exact)
    acc = torch.zeros(n, E_l.shape[0], dtype=F32)
    for k in range(dim):
        acc = fma32(a64[:, k:k + 1], e64[k][None, :], acc)
    h = -0.5 * m2
    s = torch.zeros(n, 32, dtype=F32)
    for j in range(0, dim, 32):
        w = min(32, dim - j)
        s[:, :w] = fma32(h[:, j:j + w], h[:, j:j + w], s[:, :w])
    lanes = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lanes ^ o]
    xn = s[:, 0]
    d2 = (acc + xn[:, None]) + en_l.to(F32)[None, :]
    d = torch.sqrt(torch.fmax(d2, torch.zeros((), dtype=F32)).to(F64)).to(F32)   # sqrt of fp32 in float64: correctly rounded
    return d2, d


def first_argmin(d: torch.Tensor) -> torch.Tensor:
    """Index of the first minimum along the last axis (the kernel's tie-break: the smaller index wins on equal d)."""
    m = d.min(dim=-1, keepdim=True).values
    idx = torch.arange(d.shape[-1]).expand_as(d)
    return torch.where(d == m, idx, d.shape[-1]).min(dim=-1).values


@dataclass
class Restated:
    codes: torch.Tensor       # [n, n_q] int64, frames in the order given
    resid: torch.Tensor       # [n_q, n, dim] fp32: the residual each level scored
    d2_win: torch.Tensor      # [n, n_q] fp32: the winner's d2 before the clamp
    tie: torch.Tensor         # [n, n_q] bool: another centroid has the winner's d exactly


def encode_frames(xg: torch.Tensor, E: torch.Tensor, enorm: torch.Tensor, ns: int) -> Restated:
    """Restate the encode of frames xg [n, 2, dim] (the two projected latents of each frame) through both groups:
    levels [0, ns) start from xg[:, 0], levels [ns, n_q) from xg[:, 1]."""
    n_q, bins, dim = E.shape
    n = xg.shape[0]
    codes = torch.zeros(n, n_q, dtype=torch.int64)
    resid = torch.zeros(n_q, n, dim, dtype=F32)
    d2_win = torch.zeros(n, n_q, dtype=F32)
    tie = torch.zeros(n, n_q, dtype=torch.bool)
    for g, (l0, l1) in enumerate(((0, ns), (ns, n_q))):
        r = xg[:, g].to(F32).clone()
        for l in range(l0, l1):
            if l > l0:
                r = r - E[l - 1][codes[:, l - 1]]
            resid[l] = r
            d2, d = level_distances(r, E[l], enorm[l])
            c = first_argmin(d)
            codes[:, l] = c
            d2_win[:, l] = d2.gather(1, c[:, None])[:, 0]
            tie[:, l] = (d == d.gather(1, c[:, None])).sum(dim=1) > 1
    return Restated(codes, resid, d2_win, tie)


def frame_bt(n: torch.Tensor, B: int, T: int, time_major: bool):
    """(b, t) of frame indices n: n = t * B + b (time_major) or b * T + t."""
    return (n % B, n // B) if time_major else (n // T, n % T)


def frames_of(x: torch.Tensor, ldx: int, N: int, dim: int, frames: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[n, 2, dim] latents of frames `frames` (default all N) from the flat fp32 buffer x with row stride ldx."""
    rows = x.reshape(-1).as_strided((N, 2 * dim), (ldx, 1))
    if frames is not None:
        rows = rows[frames]
    return rows.reshape(-1, 2, dim)


def encode(x: torch.Tensor, ldx: int, E: torch.Tensor, enorm: torch.Tensor, N: int, T: int, ns: int,
           time_major: bool) -> torch.Tensor:
    """rstnet_rvq_encode_f32 restated: codes int64 [B, n_q, T] of the N = B * T frames whose two latents sit at
    x[n * ldx + 0 .. 2 dim) (fp32, CPU)."""
    n_q, bins, dim = E.shape
    B = N // T
    res = encode_frames(frames_of(x, ldx, N, dim), E, enorm, ns)
    return to_layout(res.codes, torch.arange(N), B, T, time_major)


def to_layout(frame_codes: torch.Tensor, frames: torch.Tensor, B: int, T: int, time_major: bool,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Scatter [n, n_q] codes of frame indices `frames` into the [B, n_q, T] layout."""
    n_q = frame_codes.shape[1]
    if out is None:
        out = torch.full((B, n_q, T), -1, dtype=torch.int64)
    b, t = frame_bt(frames, B, T, time_major)
    out[b, :, t] = frame_codes
    return out


def gamma(n: int, u: float = U) -> float:
    return n * u / (1 - n * u)


def level_bound(r: torch.Tensor, E_l: torch.Tensor, chosen: torch.Tensor, gamma_n: float):
    """Float64 nearest-centroid bound of one level.  With d2(c) = |r - e_c|^2 in float64 and
    E_c = gamma_n (2 sum_k |r_k e_ck| + |r|^2 + |e_c|^2), a choice c* made from the fp32 sqrt distances satisfies

        d2(c*) <= min_c (d2(c) + E_c) + E_c* + 4u d2(c*)

    (the last term: sqrt rounding may merge two d2 up to 4u d2 apart, and then the smaller index wins).  Returns the
    used fraction (d2(c*) - min d2) / (bound - min d2) per frame (<= 1 when the bound holds; NaN rows give NaN) and
    whether c* is the float64 argmin."""
    r = r.to(F64)
    e = E_l.to(F64)
    rn = (r * r).sum(-1, keepdim=True)
    en = (e * e).sum(-1)[None, :]
    d2 = (rn + en - 2.0 * r @ e.T).clamp(min=0)
    S = 2.0 * r.abs() @ e.abs().T + rn + en
    Ec = gamma_n * S
    c = chosen[:, None]
    d2c, Ecc = d2.gather(1, c)[:, 0], Ec.gather(1, c)[:, 0]
    dmin = d2.min(dim=1).values
    room = (d2 + Ec).min(dim=1).values - dmin + Ecc + 4 * U * d2c
    frac = (d2c - dmin) / room
    return frac, d2c == dmin


def decisive(r: torch.Tensor, E_l: torch.Tensor, gamma_n: float) -> torch.Tensor:
    """Frames whose float64 nearest centroid b beats every other c by more than any fp32 evaluation of the distances
    can blur: d2(c) (1 - 4u) - E_c > d2(b) + E_b for all c != b.  Every chooser within `level_bound` picks b there."""
    r = r.to(F64)
    e = E_l.to(F64)
    rn = (r * r).sum(-1, keepdim=True)
    en = (e * e).sum(-1)[None, :]
    d2 = (rn + en - 2.0 * r @ e.T).clamp(min=0)
    Ec = gamma_n * (2.0 * r.abs() @ e.abs().T + rn + en)
    b = d2.argmin(dim=1, keepdim=True)
    lo = (d2 * (1 - 4 * U) - Ec).scatter(1, b, math.inf).min(dim=1).values
    return lo > (d2 + Ec).gather(1, b)[:, 0]
