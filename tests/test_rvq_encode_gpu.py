"""The codec's RVQ encoder (rstnet_rvq_encode_f32) against the exact host restatement of its fp32 arithmetic
(tests/rvq_restatement.py) and a float64 nearest-centroid bound (-m gpu).

Every case checks two things:

* bit-exact: every code equals the restatement's, with no exceptions;
* float64 bound: on the fp32 residual the kernel scored, the chosen centroid c* satisfies
  d2(c*) <= min_c (d2(c) + E_c) + E_c* + 4u d2(c*), E_c = gamma_{dim+8} (2 sum |r_k e_ck| + |r|^2 + |e_c|^2); the worst
  fraction of the bound and the share of frames where c* is the float64 argmin are printed.

The inputs put the kernel where it can go wrong: duplicated centroids where each of its argmin reductions meets them
(inside a lane's four centroids, between lanes, between CTAs, in a lane's loop over chunks) at a group's first, middle
and last level; frames exactly on a centroid (d2 cancels and may round below 0 before the clamp); an all-zero frame; a
pair of centroids whose d2 differ by one ulp while their sqrt rounds equal; a frame with a NaN component.  Codes sit in
a canvas with sentinels on both sides, the workspace is NaN bytes before every launch and is followed by guard bytes
that must stay untouched.
"""
import math
import time
from dataclasses import dataclass, field
from typing import List, Tuple

import pytest
import torch

import rvq_restatement as R
from oracle import mimi_oracle as O
from rstnet_b200 import _lib, ops
from rstnet_b200._lib import RstnetError
from test_codec_kernels_gpu import SENT, assert_canaries, canvas

pytestmark = pytest.mark.gpu
DEV, F32 = "cuda", torch.float32
RQ_BN = 128            # centroids per CTA of the level kernel (rvq.cu)
PAD = 64               # sentinel int64 slots before and after the codes


# ------------------------------------------------------------------------------------------------------------ inputs
@dataclass
class Case:
    n_q: int
    ns: int
    dim: int
    bins: int
    E: torch.Tensor                 # [n_q, bins, dim] fp32 (CPU)
    frames: torch.Tensor            # [N, 2, dim] fp32: the two projected latents of every frame
    ties: List[Tuple[int, int, int, int]] = field(default_factory=list)     # (frame, level, c1, c2), E[l][c1] == E[l][c2]
    merges: List[Tuple[int, int, int, int]] = field(default_factory=list)   # (frame, level, a, b): d2 one ulp apart, same d
    on_centroid: List[int] = field(default_factory=list)
    nan_frame: int = -1
    zero_frame: int = -1

    @property
    def enorm(self):
        return self.E.pow(2).sum(dim=-1)    # as the codec builds it (codec.py _Engine)

    def groups(self):
        return [(l0, l1) for l0, l1 in ((0, self.ns), (self.ns, self.n_q)) if l1 > l0]


def random_tables(n_q, bins, dim, seed):
    g = torch.Generator().manual_seed(seed)
    E = torch.randn(n_q, bins, dim, generator=g) * (0.75 ** torch.arange(n_q, dtype=F32))[:, None, None]
    return E


def projected_latents(N, dim, seed, proj=None):
    """Gaussian latents z [N, 512] through the two 1x1 input projections (random ones unless given)."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(N, 512, generator=g) * 1.2
    if proj is None:
        proj = [torch.randn(dim, 512, generator=g) / math.sqrt(512) for _ in range(2)]
    return torch.stack([z @ p.t() for p in proj], dim=1).contiguous()


def residual_at(case, f, level):
    """fp32 residual frame f scores at `level` under the current tables (restated)."""
    res = R.encode_frames(case.frames[f:f + 1], case.E[:level + 1], case.enorm[:level + 1], min(case.ns, level + 1))
    return res.resid[level, 0]


def pair_slots(kind, t, bins):
    """Centroid pairs placed where one reduction of the kernel meets them (t picks distinct slots):
    lane: (4j, 4j+1), one lane's four centroids;  nbr: (4j, 4j+4), j odd, so the higher lane reaches lane 0 of the
    xor butterfly first;  cta: (c, c+128), chunks k and k+1 with k odd, reduced by the next level or the finish kernel;
    loop: (c, c+32*128), chunks k and k+32, the same lane of the next level's loop over 64 chunks."""
    nch = bins // RQ_BN
    if kind == "lane":
        j = (5 + 9 * t) % 32 + 32 * (t % nch)
        return 4 * j + 1, 4 * j + 2
    if kind == "nbr":
        j = 2 * ((3 * t) % 15) + 1
        c0 = RQ_BN * (t % nch)
        return c0 + 4 * j + 3, c0 + 4 * j + 7
    if kind == "cta":
        k = 2 * (t % ((nch - 1) // 2)) + 1 if nch >= 3 else 0
        o = (37 + 5 * t) % RQ_BN
        return RQ_BN * k + o, RQ_BN * (k + 1) + o
    if kind == "loop":
        k = (3 + 5 * t) % 32
        o = (90 + 7 * t) % RQ_BN
        return RQ_BN * k + o, RQ_BN * (k + 32) + o
    raise ValueError(kind)


def build_case(n_q, ns, dim, bins, N, seed, *, E=None, proj=None, specials=True, kinds=None, merge=False):
    E = random_tables(n_q, bins, dim, seed) if E is None else E.clone()
    case = Case(n_q, ns, dim, bins, E, projected_latents(N, dim, seed + 1, proj))
    if not specials:
        return case
    g = torch.Generator().manual_seed(seed + 2)
    nch = bins // RQ_BN
    kinds = kinds or [k for k, ok in (("lane", True), ("nbr", True), ("cta", nch >= 2), ("loop", nch == 64)) if ok]
    slots = iter(torch.randperm(N, generator=g).tolist())
    used = {l: set() for l in range(n_q)}
    if merge:
        for l0, _ in case.groups():
            case.merges.append(plant_sqrt_merge(case, next(slots), l0, used[l0], g))
    # duplicated centroids at each group's first, middle and last level, planted on the residual of a frame so that
    # the pair is that frame's nearest; later levels are planted after earlier ones, whose codes they depend on
    levels = sorted({l for l0, l1 in case.groups() for l in (l0, (l0 + l1 - 1) // 2, l1 - 1)})
    for level in levels:
        for t, kind in enumerate(kinds):
            f = next(slots)
            s = 4 * t + 16 * level
            c1, c2 = pair_slots(kind, s, bins)
            while c1 in used[level] or c2 in used[level]:
                s += 1
                c1, c2 = pair_slots(kind, s, bins)
            r = residual_at(case, f, level)
            e = r + 1e-3 * r.abs().mean() * torch.randn(dim, generator=g)
            case.E[level, c1] = e
            case.E[level, c2] = e
            used[level] |= {c1, c2}
            case.ties.append((f, level, c1, c2))
    # frames exactly on a centroid: through x at each group's first level, and a centroid planted exactly on a frame's
    # residual at a later level
    for l0, l1 in case.groups():
        for _ in range(4):
            f = next(slots)
            c = int(torch.randint(0, bins, (1,), generator=g))
            while c in used[l0]:
                c = (c + 1) % bins
            case.frames[f, 0 if l0 < ns else 1] = case.E[l0, c]
            used[l0].add(c)
            case.on_centroid.append(f)
        if l1 - l0 >= 2:
            f, level = next(slots), l1 - 1
            c = next(c for c in range(7, bins) if c not in used[level])
            case.E[level, c] = residual_at(case, f, level)
            used[level].add(c)
            case.on_centroid.append(f)
    case.zero_frame = next(slots)
    case.frames[case.zero_frame] = 0
    case.nan_frame = next(slots)
    case.frames[case.nan_frame, 0, 3] = math.nan
    case.frames[case.nan_frame, 1, dim - 2] = math.nan
    return case


def plant_sqrt_merge(case, f, level, used, g):
    """Deterministic host search for centroids a < b nearest to frame f at `level` whose fp32 d2 differ by one ulp
    (d2(b) < d2(a)) while sqrtf rounds both to the same d: the kernel must keep a (first minimum of d); an argmin over
    d2 would take b.  The frame is made small against the centroids so that d2 is not a cancellation (its grid is its
    own ulp), and e_a is half a typical centroid, far nearer than the rest."""
    gi = 0 if level < case.ns else 1
    dim = case.dim
    scale = case.E[level].pow(2).sum(-1).mean().sqrt() / math.sqrt(dim)
    case.frames[f, gi] = 0.05 * scale * torch.randn(dim, generator=g)
    r = case.frames[f, gi]
    a = next(c for c in range(40, case.bins) if c not in used)
    b = next(c for c in range(a + 200, case.bins) if c not in used)
    used |= {a, b}
    # e_a such that d2(a) and the fp32 number below it have the same sqrtf (about half of all d2 do)
    e0 = 0.5 * scale * torch.randn(dim, generator=g)
    for i in range(64):
        e_a = e0 * (1 + i / 1024)
        d2_a, d_a = R.level_distances(r[None], e_a[None], e_a[None].pow(2).sum(-1))
        want = torch.nextafter(d2_a[0, 0], torch.tensor(-math.inf))
        if torch.sqrt(want.double()).float() == d_a[0, 0]:
            break
    ulp = float(d2_a[0, 0] - want)
    cands = []
    for k in range(dim):
        slope = 2 * float(e_a[k] - r[k])
        if abs(slope) < 0.5 * float(scale):
            continue
        for m in torch.linspace(0.3, 3.0, 28).tolist():
            e = e_a.clone()
            e[k] = e_a[k] - m * ulp / slope
            cands.append(e)
    C = torch.stack(cands)
    d2, d = R.level_distances(r[None], C, C.pow(2).sum(-1))
    ok = ((d2[0] == want) & (d[0] == d_a[0, 0])).nonzero()
    assert ok.numel(), "no sqrt-merge pair found"
    case.E[level, a] = e_a
    case.E[level, b] = C[int(ok[0, 0])]
    return (f, level, a, b)


# ------------------------------------------------------------------------------------------------------ restatement
_RESTATED = {}


def restate(case, key):
    if key not in _RESTATED:
        t0 = time.time()
        _RESTATED[key] = R.encode_frames(case.frames, case.E, case.enorm, case.ns)
        print(f"[rvq-encode] {key}: restated {case.frames.shape[0]} frames x {case.n_q} levels in {time.time() - t0:.1f} s")
    return _RESTATED[key]


def check_coverage(case, res):
    """The constructed inputs really produce the situations they are for."""
    for f, l, c1, c2 in case.ties:
        assert int(res.codes[f, l]) == c1 and bool(res.tie[f, l]), f"tie {c1}/{c2} at level {l} not reached (frame {f})"
    for f, l, a, b in case.merges:
        d2, d = R.level_distances(res.resid[l, f:f + 1], case.E[l], case.enorm[l])
        assert int(res.codes[f, l]) == a and d[0, a] == d[0, b] and d2[0, b] < d2[0, a] and int(d2[0].argmin()) == b, \
            f"sqrt-merge pair {a}/{b} at level {l} not reached"
    if case.on_centroid:
        assert bool((res.d2_win[case.on_centroid] < 0).any()), "no on-centroid frame has d2 below 0 before the clamp"
    if case.nan_frame >= 0:
        assert int(res.codes[case.nan_frame].abs().sum()) == 0


def check_bound(name, case, res, frames=None):
    frames = torch.arange(res.codes.shape[0]) if frames is None else frames
    worst, hits, total = 0.0, 0, 0
    for l in range(case.n_q):
        r = res.resid[l, frames]
        ok = torch.isfinite(r).all(dim=1)
        frac, is_min = R.level_bound(r[ok], case.E[l], res.codes[frames, l][ok], R.gamma(case.dim + 8))
        bad = ~(frac <= 1)
        assert not bool(bad.any()), f"{name}: level {l}: {int(bad.sum())} frames outside the float64 bound"
        worst = max(worst, float(frac.max()))
        hits += int(is_min.sum())
        total += int(ok.sum())
    print(f"[rvq-encode] {name}: worst {worst:.4f} of the float64 bound; c* is the float64 argmin in {hits}/{total} "
          f"(frame, level) pairs")


# ----------------------------------------------------------------------------------------------------------- launch
class Launch:
    """Device buffers of one encode: x rows of stride ldx (padding columns are sentinel NaN), the codes inside a
    sentinel canvas, the workspace NaN bytes followed by guard bytes."""

    def __init__(self, case, B, T, ldx, time_major, frames=None):
        self.case, self.B, self.T, self.ldx, self.tm = case, B, T, ldx, time_major
        N, dim = B * T, case.dim
        self.N = N
        self.x = canvas(N * ldx + 64)
        self.load(case.frames if frames is None else frames)
        self.E = case.E.to(DEV)
        self.Et = case.E.transpose(1, 2).contiguous().to(DEV)
        self.en = case.enorm.to(DEV)
        n_codes = B * case.n_q * T
        self.codes_f = canvas(2 * (n_codes + 2 * PAD))                  # int64 slots = two sentinel words each
        self.codes = self.codes_f.view(torch.int64)[PAD:PAD + n_codes]
        self.ws = ops.rvq_encode_workspace(N, case.n_q, dim, case.bins)
        assert self.ws % 4 == 0
        self.work = canvas(self.ws // 4 + self.ws // 4 + 1024)          # the workspace, then as many guard bytes again

    def load(self, frames):
        self.x[:self.N * self.ldx].view(self.N, self.ldx)[:, :2 * self.case.dim] = frames.reshape(self.N, -1).to(DEV)

    def fill_work(self):
        self.work.view(torch.int32).fill_(SENT)

    def run(self):
        c = self.case
        ops.rvq_encode(self.x, self.ldx, self.E, self.Et, self.en, self.codes, self.work, self.N, self.T, c.n_q, c.ns,
                       c.dim, c.bins, time_major=self.tm)

    def launch(self):
        self.fill_work()
        self.run()
        torch.cuda.synchronize()
        return self.codes.view(self.B, self.case.n_q, self.T).cpu()

    def check_buffers(self, name):
        n = self.codes.numel()
        assert_canaries(f"{name} codes canvas", self.codes_f, torch.arange(2 * PAD, 2 * (PAD + n), device=DEV))
        assert_canaries(f"{name} workspace guard", self.work, torch.arange(self.ws // 4, device=DEV))


def expect(res_codes, frames, B, T, tm):
    return R.to_layout(res_codes, frames, B, T, tm)


def check_exact(name, got, want):
    bad = got != want
    if bool(bad.any()):
        b, l, t = bad.nonzero()[0].tolist()
        raise AssertionError(f"{name}: {int(bad.sum())} of {want.numel()} codes differ from the restatement; first at "
                             f"b={b} level={l} t={t}: kernel {int(got[b, l, t])} restated {int(want[b, l, t])}")


def run_forms(name, case, res, forms):
    """forms: (B, T, time_major, ldx) launches over the first B*T frames of the case."""
    for B, T, tm, ldx in forms:
        N = B * T
        L = Launch(case, B, T, ldx, tm, case.frames[:N])
        assert torch.equal(R.frames_of(L.x.cpu(), ldx, N, case.dim).nan_to_num(7.0),
                           case.frames[:N].nan_to_num(7.0))
        got = L.launch()
        tag = f"{name} B={B} T={T} {'time' if tm else 'batch'}-major ldx={ldx}"
        check_exact(tag, got, expect(res.codes[:N], torch.arange(N), B, T, tm))
        L.check_buffers(tag)


# ------------------------------------------------------------------------------------------------------------- tests
@pytest.fixture(scope="module")
def product_case(official_weights):
    """The product's codec: 2048 bins x 256 dims, 8 levels, 1 semantic level, on the seeded codec weights."""
    w = official_weights
    proj = [w[f"quantizer.{p}.input_proj.weight"][:, :, 0] for p in ("rvq_first", "rvq_rest")]
    return build_case(8, 1, 256, 2048, 256, 11, E=O.codebooks(w), proj=proj, merge=True)


def test_rvq_encode_product_codec(product_case):
    """A streaming step at 256 streams (time-major) and 37 clips x 3 frames in both frame orders, each at ldx = 2 dim
    and at a padded ldx."""
    case = product_case
    res = restate(case, "product")
    check_coverage(case, res)
    forms = [(256, 1, True, 512), (256, 1, True, 524), (37, 3, False, 512), (37, 3, True, 524), (37, 3, False, 540),
             (128, 2, True, 512)]
    run_forms("product", case, res, forms)
    check_bound("product", case, res)


CONFIGS = {
    # MimiCodec() defaults: KT = 2 k-tiles (shorter than the 3-stage pipeline), nch = 32 chunks (one warp's worth)
    "mimi-4096x32": dict(n_q=8, ns=1, dim=32, bins=4096, N=64),
    # KT = 1 and nch = 64: each lane of the next level reduces two chunks
    "8192x16": dict(n_q=4, ns=2, dim=16, bins=8192, N=48),
    # nch = 1: the whole argmin inside one CTA; 32 levels in every group split (empty groups, both parities)
    "128x16-q32-ns0": dict(n_q=32, ns=0, dim=16, bins=128, N=40),
    "128x16-q32-ns1": dict(n_q=32, ns=1, dim=16, bins=128, N=40),
    "128x16-q32-ns2": dict(n_q=32, ns=2, dim=16, bins=128, N=40),
    "128x16-q32-ns32": dict(n_q=32, ns=32, dim=16, bins=128, N=40),
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_rvq_encode_configs(name):
    cfg = dict(CONFIGS[name])
    N = cfg.pop("N")
    case = build_case(**cfg, N=N, seed=100 + len(name) * 7 + cfg["ns"])
    res = restate(case, name)
    check_coverage(case, res)
    dim = case.dim
    run_forms(name, case, res, [(N // 4, 4, True, 2 * dim), (N // 4, 4, False, 2 * dim + 8), (N, 1, False, 2 * dim)])
    check_bound(name, case, res)


@pytest.mark.parametrize("B,T,tm", [(1, 1, False), (31, 1, True), (1, 32, False), (16, 2, True), (11, 3, True),
                                    (257, 1, False)])
def test_rvq_encode_frame_counts(B, T, tm):
    """N around the 32-frame tile: 1, 31, 32, 33, 257."""
    N = B * T
    case = build_case(4, 1, 32, 256, N, 300 + N, specials=False)
    if N > 2:
        case.frames[N - 1] = 0
        case.frames[N // 2, 1, 5] = math.nan
    res = restate(case, f"N={N}")
    run_forms(f"N={N}", case, res, [(B, T, tm, 64), (B, T, tm, 68)])
    check_bound(f"N={N}", case, res)


def test_rvq_encode_large_batch(official_weights):
    """257 clips x 128 frames on the product codec: sampled frames and the last 32-frame tile restated, every other
    code in range."""
    w = official_weights
    B, T = 257, 128
    N = B * T
    proj = [w[f"quantizer.{p}.input_proj.weight"][:, :, 0] for p in ("rvq_first", "rvq_rest")]
    case = build_case(8, 1, 256, 2048, N, 17, E=O.codebooks(w), proj=proj, specials=False)
    g = torch.Generator().manual_seed(5)
    frames = torch.cat([torch.randperm(N - 32, generator=g)[:40].sort().values, torch.arange(N - 32, N)])
    t0 = time.time()
    res = R.encode_frames(case.frames[frames], case.E, case.enorm, case.ns)
    print(f"[rvq-encode] large: restated {frames.numel()} frames in {time.time() - t0:.1f} s")
    for tm in (False, True):
        L = Launch(case, B, T, 512, tm)
        got = L.launch()
        assert bool(((got >= 0) & (got < case.bins)).all())
        b, t = R.frame_bt(frames, B, T, tm)
        want = res.codes
        bad = got[b, :, t] != want
        assert not bool(bad.any()), f"large {'time' if tm else 'batch'}-major: {int(bad.sum())} sampled codes differ"
        L.check_buffers(f"large tm={tm}")
    check_bound("large", case, res)


def test_rvq_encode_deterministic_and_graph_replay():
    """Two launches give identical codes; a CUDA graph captured around the launch, replayed after new frames are
    copied into its x buffer, gives the restatement's codes for the new frames."""
    case = build_case(8, 2, 32, 512, 96, 41)
    case2 = build_case(8, 2, 32, 512, 96, 42, specials=False)
    case2.E = case.E
    B, T = 24, 4
    L = Launch(case, B, T, 64, True)
    first = L.launch()
    second = L.launch()
    assert torch.equal(first, second)
    check_exact("replay: direct", first, expect(restate(case, "replay-1").codes, torch.arange(96), B, T, True))
    graph = ops.capture(L.run)
    L.load(case2.frames)
    L.fill_work()
    L.codes.fill_(-3)
    graph.replay()
    torch.cuda.synchronize()
    got = L.codes.view(B, 8, T).cpu()
    check_exact("replay: graph", got, expect(restate(case2, "replay-2").codes, torch.arange(96), B, T, True))
    L.check_buffers("replay")


# -------------------------------------------------------------------------------------------------------- refusals
def _small_launch():
    case = build_case(4, 1, 32, 256, 8, 9, specials=False)
    return Launch(case, 4, 2, 64, False)


BAD = {
    "bins % 128": dict(bins=192),
    "dim % 16": dict(dim=24),
    "N % T": dict(T=3),
    "ns < 0": dict(ns=-1),
    "ns > n_q": dict(ns=5),
    "ldx % 4": dict(ldx=66),
    "x misaligned": dict(x_off=1),
    "E misaligned": dict(E_off=1),
    "Et misaligned": dict(Et_off=1),
    "enorm misaligned": dict(en_off=1),
    "work misaligned": dict(work_off=1),
}


@pytest.mark.parametrize("what", list(BAD))
def test_rvq_encode_refusals(what):
    """Each out-of-contract call returns an error and launches nothing (offset views for the alignment checks)."""
    L = _small_launch()
    c = L.case
    p = dict(bins=c.bins, dim=c.dim, T=L.T, ns=c.ns, ldx=L.ldx, x_off=0, E_off=0, Et_off=0, en_off=0, work_off=0)
    p.update(BAD[what])
    n0 = _lib.launch_count()
    with pytest.raises(RstnetError, match="rvq_encode"):
        ops.rvq_encode(L.x[p["x_off"]:], p["ldx"], L.E.view(-1)[p["E_off"]:], L.Et.view(-1)[p["Et_off"]:],
                       L.en.view(-1)[p["en_off"]:], L.codes, L.work[p["work_off"]:], L.N, p["T"], c.n_q, p["ns"],
                       p["dim"], p["bins"])
    assert _lib.launch_count() == n0
    L.check_buffers(f"refused {what}")


@pytest.mark.parametrize("what", ["E", "q"])
def test_rvq_decode_gather_refuses_misaligned(what):
    B, T, n_q, dim, bins = 2, 3, 4, 32, 256
    E = torch.zeros(n_q * bins * dim + 4, device=DEV)
    q = torch.zeros(B * T * 2 * dim + 4, device=DEV)
    codes = torch.zeros(B, n_q, T, dtype=torch.int64, device=DEV)
    n0 = _lib.launch_count()
    with pytest.raises(RstnetError, match="rvq_decode_gather"):
        ops.rvq_decode_gather(codes, E[1:] if what == "E" else E, q[1:] if what == "q" else q, B * T, T, n_q, 1, dim, bins)
    assert _lib.launch_count() == n0
