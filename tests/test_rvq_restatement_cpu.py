"""The exact host restatement of the RVQ encoder (tests/rvq_restatement.py), checked without a GPU: its fmaf against
exact rational arithmetic, and its codes against the reference's cdist + argmin wherever float64 says the nearest
centroid is beyond any fp32 evaluation's reach."""
import math
import struct
from fractions import Fraction

import pytest
import torch
import torch.nn.functional as F

import rvq_restatement as R
from oracle import mimi_oracle as O

F32 = torch.float32


# ----------------------------------------------------------------------------------------------------------- fmaf
def f32(v: float) -> float:
    return struct.unpack("f", struct.pack("f", v))[0]


def round_f32(x: Fraction, zero_sign: float) -> float:
    """x rounded to the nearest fp32 (ties to even), subnormals and overflow included; an exact zero takes zero_sign."""
    if x == 0:
        return math.copysign(0.0, zero_sign)
    sign = -1.0 if x < 0 else 1.0
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    q = Fraction(2) ** (max(e, -126) - 23)            # spacing of fp32 numbers at |x|
    n = a / q
    k = math.floor(n)
    rem = n - k
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and k % 2 == 1):
        k += 1
    v = k * q
    if v >= Fraction(2) ** 128:
        return sign * math.inf
    return sign * float(v) if k else math.copysign(0.0, sign)


def fma_exact(a: float, b: float, c: float) -> float:
    p = Fraction(a) * Fraction(b)
    # an exact zero sum is -0 only when both addends are -0 (round to nearest)
    zero_sign = -1.0 if (p == 0 and math.copysign(1, a) * math.copysign(1, b) < 0 and math.copysign(1, c) < 0) else 1.0
    return round_f32(p + Fraction(c), zero_sign)


def bits(v: float) -> int:
    return struct.unpack("I", struct.pack("f", v))[0]


def check_triples(a, b, c):
    got = R.fma32(torch.tensor(a, dtype=F32), torch.tensor(b, dtype=F32), torch.tensor(c, dtype=F32))
    bad = []
    for i, (x, y, z) in enumerate(zip(a, b, c)):
        want = fma_exact(x, y, z)
        if bits(float(got[i])) != bits(want):
            bad.append((x, y, z, float(got[i]), want))
    assert not bad, f"{len(bad)} of {len(a)} fmaf results differ; first {bad[0]}"


def test_fma32_random_triples():
    g = torch.Generator().manual_seed(0)
    n = 2000
    a = torch.randn(n, generator=g) * 2.0 ** torch.randint(-30, 31, (n,), generator=g)
    b = torch.randn(n, generator=g) * 2.0 ** torch.randint(-30, 31, (n,), generator=g)
    c = torch.randn(n, generator=g) * 2.0 ** torch.randint(-30, 31, (n,), generator=g)
    # a share of c close to -a*b, where the sum cancels
    near = torch.rand(n, generator=g) < 0.25
    c = torch.where(near, -(a.double() * b.double()).float() * (1 + 2.0 ** -20 * torch.randn(n, generator=g)), c)
    check_triples(a.float().tolist(), b.float().tolist(), c.float().tolist())


def constructed_triples():
    """(a, b, c) where a float64 sum rounded once more to fp32 goes wrong, and the edges of the fp32 range."""
    out = []
    for s in (1.0, -1.0):
        for sh in (-20, 0, 17):
            k = 2.0 ** sh
            # exact fp32 midpoints: ties to even, downwards and upwards
            out.append((s * k, 2.0 ** -24, s * k * f32(1.0)))
            out.append((s * k, 2.0 ** -24, s * k * f32(1 + 2.0 ** -23)))
            # midpoint minus 2^-70 relative: float64 rounds onto the midpoint, the exact value is below it
            out.append((s * k * f32(2.0 ** -24 * (1 + 2.0 ** -23)), f32(1 - 2.0 ** -23), s * k * f32(1 + 2.0 ** -23)))
            # midpoint plus 2^-70 relative, sticky bit below the float64 ulp with the even neighbour below
            out.append((s * k * f32(2.0 ** -24 * (1 + 2.0 ** -23)), f32(1 + 2.0 ** -23), s * k * f32(1 + 2.0 ** -22)))
            out.append((s * k * f32(2.0 ** -25 * (1 - 2.0 ** -23)), f32(1 + 2.0 ** -23), -s * k * f32(1 + 2.0 ** -22)))
    # subnormal results, including ties at the smallest spacing
    for a_, b_, c_ in ((2.0 ** -75, 2.0 ** -70, 0.0), (3 * 2.0 ** -76, 2.0 ** -74, 0.0), (2.0 ** -75, 2.0 ** -75, 2.0 ** -149),
                       (1.5 * 2.0 ** -75, 2.0 ** -74, -2.0 ** -149), (2.0 ** -63, -2.0 ** -64, 2.0 ** -126),
                       (2.0 ** -100, 2.0 ** -60, -2.0 ** -149), (f32(1 + 2.0 ** -23) * 2.0 ** -70, 2.0 ** -80, 0.0)):
        out.append((a_, b_, c_))
    # sign changes and signed zeros
    for a_, b_, c_ in ((1.5, 2.0, -3.0), (-1.5, 2.0, 3.0), (0.0, -1.0, 0.0), (-0.0, 1.0, -0.0), (0.0, 1.0, -0.0),
                       (-0.0, -1.0, -0.0), (2.0 ** -80, -2.0 ** -80, 0.0), (2.0 ** -80, -2.0 ** -80, -0.0),
                       (f32(1 + 2.0 ** -23), f32(1 - 2.0 ** -23), -1.0), (3.0, f32(1 / 3), -1.0)):
        out.append((a_, b_, c_))
    # overflow
    out.append((2.0 ** 100, 2.0 ** 28, 0.0))
    out.append((f32(2 - 2.0 ** -23) * 2.0 ** 64, 2.0 ** 63, f32(2 - 2.0 ** -23) * 2.0 ** 102))
    return out


def test_fma32_constructed_cases():
    t = constructed_triples()
    check_triples(*[[f32(v) for v in col] for col in zip(*t)])


def test_fma32_midpoint_cases_are_real():
    """The sticky-bit triples do round differently from the float64 sum rounded to fp32: they test something."""
    t = constructed_triples()
    diff = 0
    for a, b, c in t:
        a, b, c = f32(a), f32(b), f32(c)
        naive = f32(a * b + c) if math.isfinite(a * b + c) else a * b + c
        if bits(naive) != bits(fma_exact(a, b, c)):
            diff += 1
    assert diff >= 6


# --------------------------------------------------------------------------------------------- against the reference
def compare_decisive(name, codes, ref, res, E, ns, frames):
    """codes == ref at every (frame, level) whose level is decisive in float64 and follows only decisive levels of its
    group (from the first undecided level on, the two residual paths may part)."""
    n_q, bins, dim = E.shape
    # the reference evaluates the norms in separate sums before its matmul: twice the kernel's dot-product length
    gam = R.gamma(2 * dim + 8)
    checked = 0
    for l0, l1 in ((0, ns), (ns, n_q)):
        alive = torch.ones(frames.numel(), dtype=torch.bool)
        for l in range(l0, l1):
            ok = R.decisive(res.resid[l], E[l], gam) & torch.isfinite(res.resid[l]).all(dim=1)
            alive &= ok
            bad = alive & (codes[:, l] != ref[:, l])
            assert not bool(bad.any()), f"{name}: level {l}: {int(bad.sum())} decisive frames differ from the reference"
            checked += int(alive.sum())
    print(f"[rvq-restatement] {name}: {checked} of {frames.numel() * n_q} (frame, level) codes decisive and equal")
    assert checked >= frames.numel() * n_q // 2


@pytest.mark.parametrize("time_major", [False, True])
def test_restatement_matches_reference_codec(time_major, official_weights):
    """The product codec (2048 bins x 256, 8 levels, 1 semantic) on projected Gaussian latents, through `encode`'s
    flat x with a padded row stride and both frame orders."""
    w = official_weights
    B, T, dim = 6, 4, 256
    g = torch.Generator().manual_seed(21)
    z = torch.randn(B, 512, T, generator=g) * 1.2
    xs = [F.conv1d(z, w[f"quantizer.{p}.input_proj.weight"]) for p in ("rvq_first", "rvq_rest")]
    xbt = torch.cat(xs, 1).permute(2, 0, 1) if time_major else torch.cat(xs, 1).permute(0, 2, 1)   # frame order
    ldx = 2 * dim + 12
    x = torch.full((B * T, ldx), math.nan)
    x[:, :2 * dim] = xbt.reshape(B * T, 2 * dim)
    E = O.codebooks(w)
    enorm = E.pow(2).sum(-1)
    codes = R.encode(x, ldx, E, enorm, B * T, T, 1, time_major)
    ref = O.rvq_encode(z, w)
    assert codes.shape == ref.shape == (B, 8, T)
    res = R.encode_frames(R.frames_of(x, ldx, B * T, dim), E, enorm, 1)
    n = torch.arange(B * T)
    b, t = R.frame_bt(n, B, T, time_major)
    assert torch.equal(codes[b, :, t], res.codes)
    compare_decisive(f"codec tm={time_major}", codes[b, :, t], ref[b, :, t], res, E, 1, n)


@pytest.mark.parametrize("ns", [0, 2, 5])
def test_restatement_matches_reference_levels(ns):
    """Random tables of 256 bins x 32 with 5 levels in each group split, against the reference's
    ResidualVectorQuantization.encode of each group."""
    n_q, bins, dim, N = 5, 256, 32, 48
    g = torch.Generator().manual_seed(30 + ns)
    E = torch.randn(n_q, bins, dim, generator=g) * (0.75 ** torch.arange(n_q, dtype=F32))[:, None, None]
    xg = torch.randn(N, 2, dim, generator=g)
    res = R.encode_frames(xg, E, E.pow(2).sum(-1), ns)
    ref = torch.zeros(N, n_q, dtype=torch.int64)
    for gi, (l0, l1) in enumerate(((0, ns), (ns, n_q))):
        if l1 > l0:
            ref[:, l0:l1] = O.rvq_levels_encode(xg[:, gi].t()[None], E[l0:l1])[:, 0].t()
    compare_decisive(f"levels ns={ns}", res.codes, ref, res, E, ns, torch.arange(N))


def test_restated_choices_meet_the_float64_bound():
    """The bound the GPU tests hold the kernel to is met by the restated arithmetic itself (on near-tie data too)."""
    n_q, bins, dim, N = 3, 512, 64, 64
    g = torch.Generator().manual_seed(4)
    E = torch.randn(n_q, bins, dim, generator=g) * 0.1
    x = torch.randn(N, 2, dim, generator=g) * 0.3
    x[:16, 0] = E[0, :16] + 1e-4 * torch.randn(16, dim, generator=g)
    res = R.encode_frames(x, E, E.pow(2).sum(-1), 1)
    for l in range(n_q):
        frac, _ = R.level_bound(res.resid[l], E[l], res.codes[:, l], R.gamma(dim + 8))
        assert bool((frac <= 1).all()), f"level {l}: worst {float(frac.max())}"


def test_nan_frame_codes_are_zero():
    """fmaxf(NaN, 0) = 0: a frame with a NaN component scores d = 0 everywhere, so the first index wins at every level
    of its group, and the frames beside it are untouched."""
    n_q, bins, dim = 4, 256, 32
    g = torch.Generator().manual_seed(6)
    E = torch.randn(n_q, bins, dim, generator=g)
    x = torch.randn(3, 2, dim, generator=g)
    clean = R.encode_frames(x, E, E.pow(2).sum(-1), 2)
    x[1, 0, 7] = math.nan
    res = R.encode_frames(x, E, E.pow(2).sum(-1), 2)
    assert res.codes[1, :2].tolist() == [0, 0]
    assert torch.equal(res.codes[1, 2:], clean.codes[1, 2:])
    assert torch.equal(res.codes[[0, 2]], clean.codes[[0, 2]])
