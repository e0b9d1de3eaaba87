"""Kernel-level GPU tests (-m gpu) of the Mimi codec: the fp32 kernels behind include/rstnet_b200.h called one by one and
compared element by element with a float64 evaluation of the same operation on the same fp32 inputs (or the oracle in
float64).

Two tolerance classes:

* Bit-exact, where the kernel's roundings can be restated in a few lines: the row moves, the counters, the RVQ decode
  gather, tf32_split, the depthwise transposed conv and the two degenerate convs (fmaf chains restated in float64 with
  one fp32 rounding per step; where that float64 value is an exact fp32 tie the emulation may double-round, so those
  elements are counted, reported and allowed 1 ulp).
* Per-element bound where there is a reduction:

      |out - ref64| <= 2 ulp_fp32(ref64) + slack

  GEMMs: S = |scale| (sum |a_k w_k| + |bias|) + |r| per element; slack = C0 S (3xTF32, precision 0) or C1 S (one TF32
  pass), plus 2^-21 sum |w_k| with the ex2.approx ELU as pre-activation.  A dropped a_lo * b_hi term costs about 2^-12 S,
  far outside C0 S.  The FFMA GEMM (gemm_rows_f32): gamma_K = K 2^-24 S, the worst case of a sequential fp32 sum.
  Attention: 2^-18 max |v| over the attended keys.  LayerNorm: 2^-20 (1 + |mean| / std) |w|.
  Every bounded case prints the worst fraction of its bound.

Every output lives in a larger buffer pre-filled with a sentinel NaN pattern (padding columns, gaps between n_split
blocks, rows before and after): every element outside the contract must be bit-identical after the launch.
"""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mimi_oracle as O
from rstnet_b200 import _lib, codec, ops
from rstnet_b200._lib import ACT_ELU, ACT_GELU, ACT_NONE, RstnetError

pytestmark = pytest.mark.gpu
DEV, F32, F64 = "cuda", torch.float32, torch.float64
C0 = 2.0 ** -17          # 3xTF32
C1 = 2.0 ** -9           # one TF32 pass
ELU_EX2 = 2.0 ** -21     # ex2.approx ELU, absolute
ATTN_C = 2.0 ** -18
LN_C = 2.0 ** -20
SENT = 0x7FBADBAD        # canary: a NaN no kernel writes
MASK13 = 0xFFFFE000


# ------------------------------------------------------------------------------------------------------------- helpers
def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def ulp32(x: torch.Tensor) -> torch.Tensor:
    """Spacing of fp32 numbers at |x| (float64): 2^(e-24) for |x| in [2^(e-1), 2^e), 2^-149 below the normal range."""
    x = x.to(F64)
    _, e = torch.frexp(x.abs())
    e = torch.where(x == 0, torch.full_like(e, -125), e.clamp(min=-125))
    return torch.pow(2.0, (e - 24).to(F64))


def check_bound(name, out, ref, slack):
    """|out - ref| <= 2 ulp_fp32(ref) + slack everywhere; prints the worst fraction of the bound used."""
    out, ref = out.detach().to(F64), ref.detach().to(F64)
    slack = slack.to(F64) if torch.is_tensor(slack) else torch.tensor(float(slack), dtype=F64, device=ref.device)
    err = (out - ref).abs()
    bound = 2 * ulp32(ref) + slack
    frac = torch.nan_to_num(err / bound, nan=float("inf"))
    used = float(frac.max()) if frac.numel() else 0.0
    print(f"[codec-kernels] {name}: worst {used:.4f} of the bound ({out.numel()} outputs)")
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())}/{out.numel()} outside the bound; first at {i}: out {float(out[i])!r} "
                             f"ref {float(ref[i])!r} bound {float(bound.expand_as(ref)[i])!r}")
    return used


def canvas(n: int) -> torch.Tensor:
    """fp32 device buffer of n elements, every one the sentinel bit pattern."""
    return torch.full((n,), SENT, dtype=torch.int32, device=DEV).view(F32)


def strided_index(size, shape, strides, offset):
    return torch.as_strided(torch.arange(size, device=DEV), shape, strides, offset)


def assert_canaries(name, buf: torch.Tensor, written: torch.Tensor, before: torch.Tensor = None):
    """Every element of `buf` outside the flat indices `written` is bit-identical to `before` (default: the sentinel)."""
    keep = torch.ones(buf.numel(), dtype=torch.bool, device=DEV)
    keep[written.reshape(-1)] = False
    got = buf.view(torch.int32)[keep]
    want = before.view(torch.int32)[keep] if before is not None else torch.full_like(got, SENT)
    bad = got != want
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} elements outside the output were written"


def same(a: torch.Tensor, b: torch.Tensor) -> bool:
    """torch.equal that also takes NaN == NaN."""
    a, b = a.cpu(), b.cpu()
    return a.shape == b.shape and a.dtype == b.dtype and bool(((a == b) | (a.isnan() & b.isnan())).all())


def error_flags(clear: bool) -> int:
    return int(_lib.lib().rstnet_device_error_flags(int(clear)))


def act64(v: torch.Tensor, act: int) -> torch.Tensor:
    if act == ACT_ELU:
        return torch.where(v > 0, v, torch.expm1(v))
    if act == ACT_GELU:
        return 0.5 * v * (1 + torch.special.erf(v / math.sqrt(2.0)))
    return v


def act_slack(v: torch.Tensor, act: int, slack: torch.Tensor) -> torch.Tensor:
    """propagate a pre-activation slack through the activation (|ELU'| <= 1, |GELU'| < 1.13) plus its own error"""
    if act == ACT_ELU:
        return slack + ELU_EX2
    if act == ACT_GELU:
        return 1.13 * slack + 2.0 ** -22 * (1 + v.abs())
    return slack


def fp32_fma(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor):
    """fmaf restated: the float64 sum of the exact product and c, rounded once to fp32.  Returns (result, tie) where tie
    marks float64 values exactly halfway between fp32 numbers (the one place the two roundings may differ)."""
    r = a.to(F64) * b.to(F64) + c.to(F64)
    r32 = r.to(F32)
    tie = (r - r32.to(F64)).abs() == ulp32(r32) / 2
    return r32, tie


def exact_or_tie(name, out, ref, tie):
    """out == ref bit for bit, except 1 ulp where the float64 restatement met an fp32 tie (counted)."""
    out, ref = out.cpu(), ref.cpu()
    tie = tie.cpu()
    eq = (out.view(torch.int32) == ref.view(torch.int32))
    near = ((out.to(F64) - ref.to(F64)).abs() <= ulp32(ref))
    print(f"[codec-kernels] {name}: {int(tie.sum())} of {out.numel()} outputs at an fp32 tie of the float64 restatement")
    bad = ~(eq | (tie & near))
    assert not bool(bad.any()), f"{name}: {int(bad.sum())} outputs differ; first at {tuple(bad.nonzero()[0].tolist())}"


# ============================================================================ tensor-core GEMM (rstnet_tc_gemm_*)
def rna_tf32_f64(x: np.ndarray) -> np.ndarray:
    """Round finite fp32 values to TF32 (10 explicit mantissa bits, fp32's exponent range) to nearest, ties away from
    zero, by magnitude arithmetic in float64: the quantum is 2^(e-11) for |x| in [2^(e-1), 2^e), and 2^-136 (the TF32
    spacing at the bottom of the normal range) below it.  Results above TF32's largest finite value become +-Inf;
    +-Inf stay."""
    x = x.astype(np.float64)
    ax = np.abs(x)
    _, e = np.frexp(ax)
    q = np.ldexp(1.0, np.maximum(e - 11, -136))
    with np.errstate(invalid="ignore"):
        r = np.floor(ax / q + 0.5) * q
    r = np.where(r > (2.0 - 2.0 ** -10) * 2.0 ** 127, np.inf, r)
    r = np.where(np.isinf(ax), np.inf, r)
    return np.copysign(r, x)


def tf32_split_ref(u: np.ndarray):
    """The documented split of rstnet_tf32_split_f32 on uint32 bit patterns: hi = rna_tf32(x), lo = rna_tf32(x - hi)
    with x - hi in fp32 (exact for finite x below the overflow band); NaN -> (x with the quiet bit set, top 19 bits
    kept; 0), +-Inf -> (+-Inf, 0)."""
    u = u.astype(np.uint32)
    x = u.view(np.float32)
    nan, inf = np.isnan(x), np.isinf(x)
    xf = np.where(nan | inf, np.float32(0), x)
    hi = rna_tf32_f64(xf).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        d = (xf - hi).astype(np.float32)
    lo = rna_tf32_f64(d).astype(np.float32)
    hi = np.where(inf, x, hi).astype(np.float32).view(np.uint32)
    hi = np.where(nan, (u | np.uint32(0x00400000)) & np.uint32(MASK13), hi).astype(np.uint32)
    lo = np.where(nan | inf, np.float32(0), lo).astype(np.float32).view(np.uint32)
    return hi, lo


def tf32_split_old(u: np.ndarray):
    """The bit formula the split used before NaN / Inf handling: hi = (u + 0x1000) & ~0x1FFF, lo likewise of x - hi."""
    u = u.astype(np.uint32)
    hi = (u + np.uint32(0x1000)) & np.uint32(MASK13)
    with np.errstate(invalid="ignore", over="ignore"):
        d = u.view(np.float32) - hi.view(np.float32)
    lo = (d.view(np.uint32) + np.uint32(0x1000)) & np.uint32(MASK13)
    return hi.astype(np.uint32), lo.astype(np.uint32)


def split_patterns():
    rng = np.random.default_rng(5)
    finite = rng.integers(0, 2 ** 32, 200000, dtype=np.uint64).astype(np.uint32)
    finite = finite[np.isfinite(finite.view(np.float32))]
    m = rng.integers(0, 2 ** 10, 4096, dtype=np.uint64).astype(np.uint32) << np.uint32(13)
    e = rng.integers(1, 254, 4096, dtype=np.uint64).astype(np.uint32) << np.uint32(23)
    ties = e | m | np.uint32(0x1000)                                     # low 13 bits exactly half an ulp
    carries = e | np.uint32(0x007FF000) | rng.integers(0x1000, 0x2000, 4096, dtype=np.uint64).astype(np.uint32)  # into the exponent
    sub = np.concatenate([np.arange(1, 70000, dtype=np.uint32), np.array([0x007FFFFF, 0x00001000, 0x00000FFF], np.uint32)])
    zeros = np.array([0x00000000, 0x80000000], np.uint32)
    band = np.array([0x7F7FEFFF, 0x7F7FF000, 0x7F7FFFFF, 0xFF7FF000], np.uint32)
    fin = np.concatenate([finite, ties, ties | np.uint32(0x80000000), carries, sub, sub | np.uint32(0x80000000), zeros, band])
    special = np.array([0x7FFFFFFF, 0xFFFFFFFF, 0x7FC00000, 0x7F800001, 0xFFC00000, 0x7F800000, 0xFF800000], np.uint32)
    return fin, special


def run_split(u: np.ndarray):
    x = torch.from_numpy(u.view(np.float32).copy()).to(DEV)
    hi, lo = ops.tf32_split(x)
    torch.cuda.synchronize()
    return hi.view(torch.int32).cpu().numpy().view(np.uint32), lo.view(torch.int32).cpu().numpy().view(np.uint32)


def test_tf32_split_bit_exact():
    """rstnet_tf32_split_f32 against round-to-nearest-ties-away computed in float64: exact ties, carries into the exponent, subnormals, +-0, the
    overflow band (hi = Inf, lo = -Inf) and every non-finite class.  On finite input the fixed formula is the old one,
    bit for bit."""
    fin, special = split_patterns()
    hi, lo = run_split(fin)
    hn, ln = tf32_split_ref(fin)
    ho, lo_old = tf32_split_old(fin)
    assert np.array_equal(hn, ho) and np.array_equal(ln, lo_old), "new formula changed a finite split"
    assert np.array_equal(hi, hn), f"hi differs at {np.nonzero(hi != hn)[0][:5]}"
    assert np.array_equal(lo, ln), f"lo differs at {np.nonzero(lo != ln)[0][:5]}"
    hi, lo = run_split(special)
    hn, ln = tf32_split_ref(special)
    assert np.array_equal(hi, hn) and np.array_equal(lo, ln)
    hif = hi.view(np.float32)
    # NaN -> a NaN in the 19 bits the tensor core reads; +-Inf -> (+-Inf, 0)
    assert np.isnan((hi[:5] & np.uint32(MASK13)).view(np.float32)).all()
    assert list(hif[5:]) == [np.inf, -np.inf] and (lo == 0).all()


class TcCase:
    """One launch of rstnet_tc_gemm: buffers with canaries, the plan, a float64 reference."""

    def __init__(self, prec, seed=0, *, I_out, O_out, N, Kc, taps=1, tap_di=0, tap_do=0, o_mul=1, a_i_stride=None,
                 a_o_stride=None, a_i_extent=None, a_o_extent=None, bias=False, scale=False, R=None, r_i_stride=None,
                 r_o_stride=None, r_split_stride=None, n_split=0, c_i_stride=None, c_o_stride=None, c_split_stride=None,
                 pre=ACT_NONE, post=ACT_NONE, C2=False, act2=ACT_ELU, a_special=None, w_special=None, w_hi_only=False):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.prec, self.pre, self.post, self.act2 = prec, pre, post, act2
        need_i, need_o = I_out + (taps - 1) * tap_di, (O_out - 1) * o_mul + 1 + (taps - 1) * tap_do
        a_i_extent = a_i_extent or need_i
        a_o_extent = a_o_extent or need_o
        a_i_stride = a_i_stride or Kc + 4
        a_o_stride = a_o_stride or a_i_extent * a_i_stride + 8
        a_off = 16
        na = a_off + (a_o_extent - 1) * a_o_stride + (a_i_extent - 1) * a_i_stride + Kc + 16
        A = torch.randn(na, generator=g, device=DEV)
        if a_special is not None:   # (c, i, o, bits)
            c, i, o, bits = a_special
            A.view(torch.int32)[a_off + o * a_o_stride + i * a_i_stride + c] = np.uint32(bits).view(np.int32).item()
        W = torch.randn(N, taps * Kc, generator=g, device=DEV) / math.sqrt(taps * Kc)
        if w_special is not None:   # (n, k, bits)
            n, k, bits = w_special
            W.view(torch.int32)[n, k] = np.uint32(bits).view(np.int32).item()
        W_arg, W_lo = W, None
        if w_hi_only:   # what the codec hands a precision-1 plan: the tf32_split hi part
            W_arg, _ = ops.tf32_split(W)
        J = N // n_split if n_split else 1
        ns = n_split or N
        c_i_stride = c_i_stride or ns + 4
        c_split_stride = c_split_stride if c_split_stride is not None else (I_out * c_i_stride + 8 if n_split else 0)
        c_o_stride = c_o_stride or (J * (I_out * c_i_stride + 8) + 4 if n_split else I_out * c_i_stride + 12)
        c_off = 32
        o_ = torch.arange(O_out, device=DEV).view(-1, 1, 1)
        i_ = torch.arange(I_out, device=DEV).view(1, -1, 1)
        n_ = torch.arange(N, device=DEV).view(1, 1, -1)
        col = (n_ // ns) * c_split_stride + n_ % ns if n_split else n_
        self.idx = c_off + o_ * c_o_stride + i_ * c_i_stride + col
        nc = int(self.idx.max()) + 1 + 64
        self.C = canvas(nc)
        self.C2 = canvas(nc) if C2 else None
        bias_t = torch.randn(N, generator=g, device=DEV) if bias else None
        scale_t = torch.rand(N, generator=g, device=DEV) + 0.5 if scale else None
        kw = dict(taps=taps, tap_di=tap_di, tap_do=tap_do, o_mul=o_mul, bias=bias_t, scale=scale_t, n_split=n_split,
                  c_split_stride=c_split_stride, pre_act=pre, post_act=post, precision=prec, W_lo=W_lo)
        r_vals = None
        if R == "inplace":   # R == C: the epilogue reads the residual where it writes
            r_vals = torch.randn(self.idx.shape, generator=g, device=DEV)
            self.C[self.idx] = r_vals
            kw.update(R=self.C, r_off=c_off, r_i_stride=c_i_stride, r_o_stride=c_o_stride, r_split_stride=c_split_stride)
        elif R == "sep":     # R with its own strides
            r_i_stride = r_i_stride or ns + 8
            r_split_stride = r_split_stride if r_split_stride is not None else (I_out * r_i_stride + 4 if n_split else 0)
            r_o_stride = r_o_stride or (J * (I_out * r_i_stride + 4) + 8 if n_split else I_out * r_i_stride + 16)
            rcol = (n_ // ns) * r_split_stride + n_ % ns if n_split else n_
            ridx = 8 + o_ * r_o_stride + i_ * r_i_stride + rcol
            Rb = torch.randn(int(ridx.max()) + 64, generator=g, device=DEV)
            r_vals = Rb[ridx]
            kw.update(R=Rb, r_off=8, r_i_stride=r_i_stride, r_o_stride=r_o_stride, r_split_stride=r_split_stride)
        if C2:
            kw.update(C2=self.C2, c2_off=c_off, act2=act2)
        self.C_before = self.C.clone()
        self.plan = ops.TcGemm(A, a_off, a_i_stride, a_o_stride, Kc, a_i_extent, a_o_extent, W_arg, Kc, self.C, c_off,
                               c_i_stride, c_o_stride, I_out, O_out, **kw)
        # ---- float64 reference of the same contraction (TMA zero fill past the extents)
        A64 = torch.zeros(max(need_o, a_o_extent), max(need_i, a_i_extent), Kc, dtype=F64, device=DEV)
        A64[:a_o_extent, :a_i_extent] = torch.as_strided(A, (a_o_extent, a_i_extent, Kc), (a_o_stride, a_i_stride, 1), a_off).to(F64)
        A64 = act64(A64, pre)
        W64 = W.to(F64)
        acc = torch.zeros(O_out, I_out, N, dtype=F64, device=DEV)
        S = torch.zeros_like(acc)
        exact_ieee = a_special is not None or w_special is not None
        for t in range(taps):
            At = A64[torch.arange(O_out, device=DEV) * o_mul + t * tap_do][:, torch.arange(I_out, device=DEV) + t * tap_di]
            Wt = W64[:, t * Kc:(t + 1) * Kc]
            if exact_ieee:   # IEEE Inf / NaN arithmetic element by element (a BLAS may not keep it)
                acc += (At.unsqueeze(2) * Wt).sum(-1)
                fin_a = torch.nan_to_num(At, nan=0.0, posinf=0.0, neginf=0.0)
                fin_w = torch.nan_to_num(Wt, nan=0.0, posinf=0.0, neginf=0.0)
                S += fin_a.abs() @ fin_w.abs().t()
            else:
                acc += At @ Wt.t()
                S += At.abs() @ Wt.abs().t()
        c = C0 if prec == 0 else C1
        slack = c * S
        if pre == ACT_ELU:
            slack = slack + ELU_EX2 * torch.nan_to_num(W64, posinf=0.0, neginf=0.0, nan=0.0).abs().sum(1)
        v = acc
        if bias:
            v = v + bias_t.to(F64)
            slack = slack + c * bias_t.to(F64).abs()
        if scale:
            v = v * scale_t.to(F64)
            slack = slack * scale_t.to(F64)
        if r_vals is not None:
            v = v + r_vals.to(F64)
            slack = slack + c * r_vals.to(F64).abs()
        self.v, self.slack = v, slack
        self.ref = act64(v, post)
        self.ref_slack = act_slack(v, post, slack)
        if C2:
            self.ref2 = act64(v, act2)
            self.ref2_slack = act_slack(v, act2, slack)

    def run(self):
        self.plan.run()
        torch.cuda.synchronize()
        return self.C[self.idx]

    def check(self, name):
        out = self.run()
        used = check_bound(name, out, self.ref, self.ref_slack)
        assert_canaries(name, self.C, self.idx)
        if self.C2 is not None:
            used = max(used, check_bound(name + " C2", self.C2[self.idx], self.ref2, self.ref2_slack))
            assert_canaries(name + " C2", self.C2, self.idx)
        return used


TC_FEATURES = {
    "I1": dict(I_out=1, O_out=1, N=64, Kc=32),
    "I127": dict(I_out=127, O_out=1, N=28, Kc=96),
    "I128_Kc160": dict(I_out=128, O_out=1, N=36, Kc=160),            # 5 stages: not a whole promotion chunk
    "I129_Kc1024": dict(I_out=129, O_out=1, N=60, Kc=1024),
    "tiles_per_sm": dict(I_out=20000, O_out=1, N=128, Kc=64),        # > 2 tiles per persistent CTA
    "N4": dict(I_out=200, O_out=2, N=4, Kc=32),
    "N68": dict(I_out=130, O_out=1, N=68, Kc=32),
    "N1028": dict(I_out=100, O_out=1, N=1028, Kc=64),
    "conv_s4_k8": dict(I_out=40, O_out=5, N=64, Kc=32, taps=8, tap_do=1, o_mul=4),
    "conv_s8_k16": dict(I_out=130, O_out=3, N=32, Kc=32, taps=16, tap_do=1, o_mul=8),
    "conv_s1_k3_omul1": dict(I_out=64, O_out=7, N=64, Kc=64, taps=3, tap_do=1, o_mul=1),
    "omul2_k1": dict(I_out=70, O_out=4, N=36, Kc=32, o_mul=2),
    "taps_di": dict(I_out=200, O_out=2, N=68, Kc=32, taps=3, tap_di=1),   # taps along i (batch-major conv)
    "taps_di2": dict(I_out=129, O_out=1, N=32, Kc=64, taps=2, tap_di=3),
    "bias": dict(I_out=150, O_out=2, N=64, Kc=64, bias=True),
    "scale": dict(I_out=150, O_out=2, N=64, Kc=64, scale=True),
    "R_sep": dict(I_out=150, O_out=2, N=64, Kc=64, R="sep"),
    "R_inplace": dict(I_out=150, O_out=2, N=64, Kc=64, R="inplace"),
    "bias_scale_R": dict(I_out=150, O_out=2, N=96, Kc=96, bias=True, scale=True, R="sep"),
    "bias_scale_Rinplace": dict(I_out=300, O_out=1, N=512, Kc=128, bias=True, scale=True, R="inplace"),
    "post_elu": dict(I_out=150, O_out=2, N=64, Kc=64, bias=True, post=ACT_ELU),
    "post_gelu": dict(I_out=150, O_out=2, N=128, Kc=64, bias=True, post=ACT_GELU),
    "C2": dict(I_out=150, O_out=2, N=64, Kc=64, bias=True, C2=True),
    "C2_post_gelu": dict(I_out=150, O_out=1, N=64, Kc=64, bias=True, C2=True, post=ACT_GELU, act2=ACT_ELU),
    "nsplit_C2": dict(I_out=130, O_out=3, N=128, Kc=64, taps=2, tap_do=1, bias=True, n_split=32, C2=True),
    "nsplit_R": dict(I_out=130, O_out=2, N=96, Kc=64, taps=2, tap_do=1, bias=True, n_split=24, R="sep"),
    "nsplit_R_post": dict(I_out=64, O_out=2, N=256, Kc=32, n_split=64, R="sep", post=ACT_ELU, scale=True),
    # the A box reads past the extents: TMA fills zeros
    "past_i_extent": dict(I_out=200, O_out=1, N=64, Kc=32, taps=3, tap_di=1, a_i_extent=190),
    "past_o_extent": dict(I_out=40, O_out=5, N=64, Kc=32, taps=4, tap_do=1, o_mul=2, a_o_extent=9),
}


@pytest.mark.parametrize("name", list(TC_FEATURES))
@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("pre", [ACT_NONE, ACT_ELU])
def test_tc_gemm_features(name, prec, pre):
    case = TcCase(prec, seed=zlib.crc32(name.encode()) % 1000 + 7 * prec + pre, pre=pre, **TC_FEATURES[name])
    case.check(f"tc {name} prec={prec} pre={pre}")


def expected_bn(I_out, O_out, N, n_sms):
    """rstnet_tc_gemm_create's tile width: 64 for N >= 64, narrowed to 32 when that takes at most 1.5x the rounds of the
    SMs (a BN = 64 tile costs about 1.5 BN = 32 tiles)."""
    bn = 64 if N >= 64 else 32
    mt = -(-I_out // 128) * O_out
    t64, t32 = mt * -(-N // 64), mt * -(-N // 32)
    if bn == 64 and -(-t32 // n_sms) * 2 <= -(-t64 // n_sms) * 3:
        bn = 32
    return bn


def plan_grid(plan):
    gx, gy, bn = C.c_int32(), C.c_int32(), C.c_int32()
    assert _lib.lib().rstnet_tc_gemm_grid(plan._h, C.byref(gx), C.byref(gy), C.byref(bn)) == 0
    return gx.value, gy.value, bn.value


def test_tc_gemm_tile_choice():
    n = sms()
    shapes = [(128, 1, 64), (128 * n, 1, 64), (128 * n, 1, 128), (256, 256, 64), (129, 1, 1024), (128 * 3 * n, 1, 256),
              (300, 1, 32), (40, 5, 64), (128 * n // 2, 1, 128)]
    seen = set()
    for I, O_, N in shapes:
        case = TcCase(1, I_out=I, O_out=O_, N=N, Kc=32)
        gx, gy, bn = plan_grid(case.plan)
        assert bn == expected_bn(I, O_, N, n), (I, O_, N, bn)
        assert gx == -(-I // 128) * O_ and gy == -(-N // bn)
        seen.add(bn)
        if I * O_ * N <= 128 * n * 128:
            case.check(f"tc tile I={I} O={O_} N={N} bn={bn}")
    assert seen == {32, 64}


def raw_desc(**over):
    A = torch.zeros(4096, device=DEV)
    W = torch.zeros(64, 64, device=DEV)
    Cb = torch.zeros(4096, device=DEV)
    d = _lib.TcGemmDesc()
    d.A, d.a_i_stride, d.a_o_stride, d.a_c_extent, d.a_i_extent, d.a_o_extent = A.data_ptr(), 64, 64 * 32, 64, 32, 1
    d.taps, d.tap_di, d.tap_do, d.o_mul = 1, 0, 0, 1
    d.W, d.W_lo, d.N, d.Kc, d.I_out, d.O_out = W.data_ptr(), W.data_ptr(), 64, 64, 32, 1
    d.C, d.c_i_stride, d.c_o_stride = Cb.data_ptr(), 64, 64 * 32
    d.precision = 0
    for k, v in over.items():
        setattr(d, k, v)
    return d, (A, W, Cb)


@pytest.mark.parametrize("over,msg", [
    (dict(Kc=48, a_c_extent=48), "Kc (48) must be a multiple of 32"),
    (dict(N=30), "N (30) must be a multiple of 4"),
    (dict(a_i_stride=66), "16-byte alignment"),
    (dict(c_i_stride=70), "16-byte alignment"),
    (dict(n_split=6), "16-byte alignment"),
    ("A+4", "16-byte alignment"),
    ("C+4", "16-byte alignment"),
    (dict(pre_act=ACT_GELU), "pre_act must be NONE or ELU"),
    (dict(precision=2), "precision must be 0"),
    (dict(W_lo=None), "precision 0 (3xTF32) needs W_lo"),
])
def test_tc_gemm_create_refusals(over, msg):
    if isinstance(over, str):
        d, keep = raw_desc()
        if over == "A+4":
            d.A = d.A + 4
        else:
            d.C = d.C + 4
    else:
        d, keep = raw_desc(**over)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    h = C.c_void_p()
    rc = _lib.lib().rstnet_tc_gemm_create(C.byref(d), C.byref(h))
    assert rc != 0 and not h.value
    assert msg in _lib.lib().rstnet_last_error().decode()
    assert _lib.launch_count() == n0


SPECIALS = {"nan_cuda": 0x7FFFFFFF, "nan_neg": 0xFFFFFFFF, "nan_torch": 0x7FC00000, "nan_snan": 0x7F800001,
            "pinf": 0x7F800000, "ninf": 0xFF800000}


@pytest.mark.parametrize("where,pre", [("A", ACT_NONE), ("A", ACT_ELU), ("W", ACT_NONE)])   # pre_act applies to A only
@pytest.mark.parametrize("special", list(SPECIALS))
@pytest.mark.parametrize("prec", [0, 1])
def test_tc_gemm_nonfinite(where, pre, special, prec):
    """A NaN / Inf at one (c, i, o) of A, or in one weight: exactly the outputs whose float64 result is non-finite are
    non-finite, with the same class; every other output stays within the bound.  ELU(-Inf) = -1 is finite."""
    bits = SPECIALS[special]
    spec = dict(I_out=130, O_out=2, N=64, Kc=64, taps=2, tap_di=1, pre=pre, w_hi_only=prec == 1)
    if where == "A":
        spec["a_special"] = (37, 128, 1, bits)     # row 128: the second i tile, taps reach it from rows 127 and 128
    else:
        spec["w_special"] = (5, 64 + 17, bits)
    case = TcCase(prec, seed=bits % 9973, **spec)
    out = case.run()
    ref = case.ref
    nf_ref, nf_out = ~torch.isfinite(ref), ~torch.isfinite(out)
    assert torch.equal(nf_ref, nf_out), f"non-finite outputs: {int(nf_out.sum())} vs float64 {int(nf_ref.sum())}"
    if nf_ref.any():
        assert torch.equal(ref.isnan(), out.isnan()) or (where == "W" and prec == 0 and bits in (0x7F800000, 0xFF800000)), \
            "NaN class differs"
        inf = ref.isinf()
        if where == "W" and prec == 0 and bits in (0x7F800000, 0xFF800000):
            # documented: an infinite weight at precision 0 may give NaN where the float64 result is +-Inf
            assert bool((out[inf].isnan() | (out[inf] == ref[inf].to(F32))).all())
        else:
            assert torch.equal(out[inf], ref[inf].to(F32)), "Inf sign differs"
    fin = torch.isfinite(ref)
    check_bound(f"tc nonfinite {where} {special} prec={prec} pre={pre} (finite part)", out[fin], ref[fin],
                case.ref_slack[fin])
    assert_canaries("tc nonfinite", case.C, case.idx)


# ---- every descriptor the codec builds, replayed in isolation
def _record_codec_descriptors(monkeypatch, official_weights):
    recs = []
    real = ops.TcGemm

    class Recording(real):
        def __init__(self, *a, **kw):
            recs.append((a, kw))
            super().__init__(*a, **kw)

    monkeypatch.setattr(ops, "TcGemm", Recording)
    m = codec.MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(official_weights, strict=True)
    m = m.to(DEV).eval()
    eng = m._eng()
    configs = []
    for B in (256, 3):
        act = torch.ones(B, dtype=torch.int64, device=DEV)
        configs.append(lambda B=B, act=act: codec._EncPlan(eng, B, m.frame_size, True, True, active=act))
        configs.append(lambda B=B, act=act: codec._DecPlan(eng, B, 1, True, True, active=act))
    configs.append(lambda: codec._EncPlan(eng, 128, 2 * m.frame_size, False, True))
    configs.append(lambda: codec._DecPlan(eng, 128, 2, False, True))

    def dec_prec1():
        m.decoder_precision = 1
        try:
            return codec._DecPlan(eng, 3, 1, True, True, active=torch.ones(3, dtype=torch.int64, device=DEV))
        finally:
            m.decoder_precision = 0
    configs.append(dec_prec1)
    specs = {}
    for make in configs:
        n0 = len(recs)
        plan = make()
        del plan
        for a, kw in recs[n0:]:
            (A, a_off, a_i_stride, a_o_stride, a_c_extent, a_i_extent, a_o_extent, W, Kc, C_, c_off, c_i_stride, c_o_stride,
             I_out, O_out) = a
            R = kw.get("R")
            r = None if R is None else ("inplace" if R.data_ptr() == C_.data_ptr() and kw.get("r_off", 0) == c_off else "sep")
            spec = dict(I_out=I_out, O_out=O_out, N=W.shape[0], Kc=Kc, taps=kw.get("taps", 1), tap_di=kw.get("tap_di", 0),
                        tap_do=kw.get("tap_do", 0), o_mul=kw.get("o_mul", 1), a_i_stride=a_i_stride, a_o_stride=a_o_stride,
                        a_i_extent=a_i_extent, a_o_extent=a_o_extent, bias=kw.get("bias") is not None,
                        scale=kw.get("scale") is not None, R=r, n_split=kw.get("n_split", 0), c_i_stride=c_i_stride,
                        c_o_stride=c_o_stride, c_split_stride=kw.get("c_split_stride", 0), pre=kw.get("pre_act", ACT_NONE),
                        post=kw.get("post_act", ACT_NONE), C2=kw.get("C2") is not None, act2=kw.get("act2", ACT_NONE))
            assert a_c_extent == Kc
            if r == "sep":
                spec.update(r_i_stride=kw["r_i_stride"], r_o_stride=kw["r_o_stride"], r_split_stride=kw.get("r_split_stride", 0))
            key = (kw.get("precision", 0),) + tuple(sorted(spec.items()))
            specs[key] = (kw.get("precision", 0), spec)
    monkeypatch.setattr(ops, "TcGemm", real)
    return list(specs.values())


def test_tc_gemm_codec_descriptors(monkeypatch, official_weights):
    """Every tensor-core descriptor of the streaming plans at B = 256 and B = 3 (and the precision-1 decoder), and of the
    non-streaming plans at B = 128, on fresh random buffers of the recorded extents, against float64."""
    specs = _record_codec_descriptors(monkeypatch, official_weights)
    assert len(specs) >= 20
    worst = 0.0
    for k, (prec, spec) in enumerate(specs):
        case = TcCase(prec, seed=k, **spec)
        worst = max(worst, case.check(f"codec descriptor {k} prec={prec} " + " ".join(
            f"{a}={spec[a]}" for a in ("I_out", "O_out", "N", "Kc", "taps", "o_mul", "n_split", "R", "C2", "pre", "post"))))
        del case
        torch.cuda.empty_cache()
    print(f"[codec-kernels] {len(specs)} distinct codec descriptors, worst {worst:.4f} of the bound")


# ============================================================================ FFMA GEMM (rstnet_gemm_rows_f32)
def rows_cfg(M, N, n_sms):
    """rstnet_gemm_rows_f32's tile choice: the widest tile that still gives >= 2 CTAs per SM."""
    ctas = lambda bm, bn: -(-M // bm) * -(-N // bn)
    want = 2 * n_sms
    if N <= 32:
        return "128x32" if ctas(128, 32) >= want else "32x32/narrow"
    if N <= 64:
        if ctas(128, 64) >= want:
            return "128x64/N64"
        return "64x64/N64" if ctas(64, 64) >= want else "32x64/N64"
    for bm, bn in ((128, 128), (128, 64), (64, 64), (32, 64)):
        if ctas(bm, bn) >= want:
            return f"{bm}x{bn}"
    return "32x32"


def rows_case(name, batch, rows, N, K, *, taps=1, time_major=False, pre=ACT_NONE, post=ACT_NONE, bias=False, scale=False,
              R=False, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    kc = K // taps
    if time_major:   # batch = output time steps, rows = streams; tap j of a row is one time step (rows * kc) further on
        a_bs, a_rs, tap_stride = rows * kc, kc, rows * kc
    else:            # rows of a stream overlap (a conv window) with a padded row stride
        a_bs, a_rs, tap_stride = (rows + 8) * (K + 4), K + 4, 0
    a_off = 4
    na = a_off + (batch - 1) * a_bs + (rows - 1) * a_rs + (taps - 1) * tap_stride + K + 16
    A = torch.randn(na, generator=g, device=DEV)
    Wt = torch.randn(K, N, generator=g, device=DEV) / math.sqrt(K)
    c_rs, c_bs = N + 4, rows * (N + 4) + 8
    c_off = 16
    idx = strided_index(c_off + batch * c_bs + 64, (batch, rows, N), (c_bs, c_rs, 1), c_off)
    Cb = canvas(c_off + batch * c_bs + 64)
    bias_t = torch.randn(N, generator=g, device=DEV) if bias else None
    scale_t = torch.rand(N, generator=g, device=DEV) + 0.5 if scale else None
    kw = dict(bias=bias_t, scale=scale_t, pre_act=pre, post_act=post, taps=taps, tap_stride=tap_stride)
    r_vals = None
    if R:
        r_bs, r_rs = rows * (N + 12) + 4, N + 12
        Rb = torch.randn(8 + batch * r_bs + 64, generator=g, device=DEV)
        r_vals = torch.as_strided(Rb, (batch, rows, N), (r_bs, r_rs, 1), 8)
        kw.update(R=Rb, r_off=8, r_bs=r_bs, r_rs=r_rs)
    ops.gemm_rows(A, a_off, a_bs, a_rs, Wt, Cb, c_off, c_bs, c_rs, batch, rows, **kw)
    torch.cuda.synchronize()
    parts = [torch.as_strided(A, (batch, rows, kc), (a_bs, a_rs, 1), a_off + j * tap_stride) for j in range(taps)] \
        if taps > 1 else [torch.as_strided(A, (batch, rows, K), (a_bs, a_rs, 1), a_off)]
    a64 = act64(torch.cat(parts, -1).to(F64), pre)
    w64 = Wt.to(F64)
    v, S = a64 @ w64, a64.abs() @ w64.abs()
    if bias:
        v, S = v + bias_t.to(F64), S + bias_t.to(F64).abs()
    if scale:
        v, S = v * scale_t.to(F64), S * scale_t.to(F64)
    if R:
        v, S = v + r_vals.to(F64), S + r_vals.to(F64).abs()
    slack = K * 2.0 ** -24 * S + (2.0 ** -22 * w64.abs().sum(0) if pre == ACT_ELU else 0.0)
    used = check_bound(name, Cb[idx], act64(v, post), act_slack(v, post, slack) if post != ACT_ELU else slack + 2.0 ** -22)
    assert_canaries(name, Cb, idx)
    return used


@pytest.mark.parametrize("target,N,K", [("128x32", 32, 64), ("32x32/narrow", 28, 96), ("128x64/N64", 64, 64),
                                        ("64x64/N64", 60, 96), ("32x64/N64", 36, 64), ("128x128", 256, 64),
                                        ("128x64", 128, 96), ("64x64", 128, 64), ("32x64", 132, 64), ("32x32", 68, 64)])
def test_gemm_rows_tile_configs(target, N, K):
    """Each branch of the launcher's tile choice, forced by (M, N) from the SM count; ragged M and N, canaries."""
    n = sms()
    M = {"128x32": 128 * 2 * n + 5, "128x64/N64": 128 * 2 * n + 3, "64x64/N64": 64 * 2 * n - 1, "128x128": 128 * n + 7,
         "128x64": 128 * n - 3, "64x64": 64 * n + 1, "32x64": 32 * n + 3}.get(target, 37)
    assert rows_cfg(M, N, n) == target, (M, N, rows_cfg(M, N, n))
    rows = 7 if M % 7 == 0 else 1
    rows_case(f"gemm_rows {target} M={M} N={N}", M // rows, rows, N, K, bias=True, seed=N + K)


@pytest.mark.parametrize("variant", ["taps_tm", "taps_tm_elu", "R_scale", "pre_elu_post_gelu", "post_elu"])
def test_gemm_rows_features(variant):
    if variant.startswith("taps_tm"):   # the time-major fallback of the tensor-core plans: taps B * Cin apart
        rows_case(f"gemm_rows {variant}", 12, 37, 64, 3 * 64, taps=3, time_major=True, bias=True,
                  pre=ACT_ELU if variant.endswith("elu") else ACT_NONE, post=ACT_ELU, seed=3)
    elif variant == "R_scale":
        rows_case("gemm_rows R + scale", 5, 41, 100, 128, bias=True, scale=True, R=True, seed=4)
    elif variant == "pre_elu_post_gelu":
        rows_case("gemm_rows pre ELU post GELU", 3, 50, 72, 96, pre=ACT_ELU, post=ACT_GELU, seed=5)
    else:
        rows_case("gemm_rows post ELU", 2, 77, 44, 32, bias=True, post=ACT_ELU, seed=6)


# ============================================================================ ring attention
def ring_reference(q, K, V, off, T, cap, context, linear):
    """q [B,H,T,D], ring K/V [B,H,cap,D] (float64), per-stream offsets -> out [B,T,H,D] and the per-query slack."""
    B, H, _, D = q.shape
    out = torch.zeros(B, T, H, D, dtype=F64)
    slack = torch.zeros(B, T, H, D, dtype=F64)
    for b in range(B):
        end = int(off[b]) + T
        slots = torch.arange(cap)
        if linear:
            pos_k = slots
        else:   # the slot labels of RingKVCache.complete after this step's T positions (the oracle's KVRing)
            ring = O.KVRing(1, 1, 1, cap, dtype=F64)
            ring.end_offset = end - T
            _, _, pos_k = ring.complete(torch.zeros(1, 1, T, 1, dtype=F64), torch.zeros(1, 1, T, 1, dtype=F64))
        for t in range(T):
            pq = int(off[b]) + t
            m = (pos_k >= 0) & (pq - pos_k >= 0) & (pq - pos_k < context)
            s = torch.einsum("hd,hkd->hk", q[b, :, t], K[b]) / math.sqrt(D)
            s = s.masked_fill(~m, float("-inf"))
            p = torch.softmax(s, -1)
            out[b, t] = torch.einsum("hk,hkd->hd", p, V[b])
            vmax = V[b][:, m].abs().amax(dim=(1, 2)) if bool(m.any()) else torch.zeros(H, dtype=F64)
            slack[b, t] = ATTN_C * vmax[:, None]
    return out, slack


@pytest.mark.parametrize("name,T,D,cap,context,offs,layout,qpad", [
    ("T1", 1, 64, 16, 250, [0, 5, 40, 3], "bm", 0),
    ("T1_D32_tc", 1, 32, 10, 8, [9, 10, 33, 2], "tc", 0),
    ("generic_D32", 2, 32, 16, 16, [0, 7, 30, 15], "bm", 0),
    ("generic_D128_T3", 3, 128, 12, 250, [0, 4, 20, 100], "bm", 0),
    ("generic_D64_unaligned", 2, 64, 16, 250, [1, 14, 31, 2], "bm", 2),
    ("generic_D64_T5_unaligned", 5, 64, 24, 10, [0, 19, 40, 3], "tc", 1),
    ("pair64", 2, 64, 250, 250, [0, 100, 248, 500], "bm", 0),
    ("pair64_T3_wrap", 3, 64, 16, 250, [0, 13, 14, 45], "bm", 0),
    ("pair64_T5_ctx_lt_cap", 5, 64, 40, 12, [2, 35, 80, 1], "tc", 0),
    ("pair64_tc_layout", 2, 64, 250, 250, [10, 249, 251, 0], "tc", 0),
])
def test_ring_attention(name, T, D, cap, context, offs, layout, qpad):
    """rstnet_ring_attention_f32, all three kernels (T = 1; generic pair: D != 64 or unaligned strides; pair64), per-stream
    offsets (some rings wrapped, including the masked oldest slot), batch-major and tensor-core layouts, context < cap.
    The ring is left bit-identical; output canaries."""
    B, H = len(offs), 3
    g = torch.Generator().manual_seed(T * 131 + D + cap)
    qkv = torch.randn(T, B, 3 * H * D, generator=g) * 0.6
    K = torch.randn(B, H, cap, D, generator=g) * 0.6
    V = torch.randn(B, H, cap, D, generator=g)
    row = 3 * H * D + qpad
    if layout == "tc":    # [T, B, 3HD]: q_ts = B * 3HD
        q_bs, q_ts, o_bs, o_ts = row, B * row, H * D, B * H * D
        qbuf = torch.zeros(T * B * row + 8)
        qbuf[:T * B * row].view(T, B, row)[..., :3 * H * D] = qkv
    else:                 # [B, T, 3HD]
        q_bs, q_ts, o_bs, o_ts = T * row, row, T * H * D, H * D
        qbuf = torch.zeros(T * B * row + 8)
        qbuf[:T * B * row].view(B, T, row)[..., :3 * H * D] = qkv.transpose(0, 1)
    qd = qbuf.to(DEV)
    kv = torch.stack([K, V]).contiguous().to(DEV)
    kv0 = kv.clone()
    off = torch.tensor(offs, dtype=torch.int64)
    offd = off.to(DEV)
    n_out = T * B * H * D
    out = canvas(n_out + 64)
    out_v = out[16:16 + n_out]
    ops.ring_attention(qd, q_bs, q_ts, kv, offd, out_v, o_bs, o_ts, B, T, H, D, cap, context, False)
    torch.cuda.synchronize()
    q = qkv[..., :H * D].view(T, B, H, D).permute(1, 2, 0, 3).to(F64)
    ref, slack = ring_reference(q, K.to(F64), V.to(F64), off, T, cap, context, False)
    if layout == "tc":
        got = out_v.view(T, B, H, D).transpose(0, 1).cpu()
    else:
        got = out_v.view(B, T, H, D).cpu()
    check_bound(f"ring_attention {name}", got, ref, slack)
    assert torch.equal(kv, kv0), "ring_attention wrote the ring"
    assert_canaries(f"ring_attention {name}", out, torch.arange(16, 16 + n_out, device=DEV))


def test_ring_attention_linear():
    """linear != 0 (non-streaming KVCacheResult.from_kv): every position in [0, cap) attendable, context mask only."""
    B, H, T, D, cap, context = 2, 2, 40, 64, 40, 16
    g = torch.Generator().manual_seed(9)
    qkv = torch.randn(B, T, 3 * H * D, generator=g) * 0.6
    K = torch.randn(B, H, cap, D, generator=g) * 0.6
    V = torch.randn(B, H, cap, D, generator=g)
    out = torch.empty(B, T, H * D, device=DEV)
    kv = torch.stack([K, V]).contiguous().to(DEV)
    for T_ in (T, 1):   # pair64 and the T = 1 kernel
        off = torch.zeros(1, dtype=torch.int64)
        ops.ring_attention(qkv.to(DEV).contiguous(), T * 3 * H * D, 3 * H * D, kv, off.to(DEV), out, T * H * D, H * D, B, T_, H,
                           D, cap, context, True)
        torch.cuda.synchronize()
        q = qkv[:, :T_, :H * D].reshape(B, T_, H, D).permute(0, 2, 1, 3).to(F64)
        ref, slack = ring_reference(q, K.to(F64), V.to(F64), torch.zeros(B, dtype=torch.int64), T_, cap, context, True)
        check_bound(f"ring_attention linear T={T_}", out.view(B, T, H, D)[:, :T_].cpu(), ref, slack)


# ============================================================================ RVQ
def _rvq_tables(w):
    E = O.codebooks(w)
    return E, E.to(DEV), E.transpose(1, 2).contiguous().to(DEV), E.pow(2).sum(-1).to(DEV)


@pytest.mark.parametrize("B,T", [(256, 2), (37, 3)])
def test_rvq_encode_time_major(B, T, official_weights):
    """time_major = 1 (the streaming tensor-core plans: frame n = t * B + b) against the oracle; indices equal wherever the
    float64 margin is above 1e-4."""
    w = official_weights
    cd, n_q, bins = 256, 8, 2048
    g = torch.Generator().manual_seed(B + T)
    z = torch.randn(B, 512, T, generator=g) * 1.2
    x1 = F.conv1d(z, w["quantizer.rvq_first.input_proj.weight"])
    x2 = F.conv1d(z, w["quantizer.rvq_rest.input_proj.weight"])
    xproj = torch.cat([x1, x2], 1).permute(2, 0, 1).reshape(T * B, 2 * cd).contiguous()   # [T, B, 2cd]
    E, Ed, Et, en = _rvq_tables(w)
    codes = torch.full((B, n_q, T), -7, dtype=torch.int64, device=DEV)
    work = torch.empty(ops.rvq_encode_workspace(B * T, n_q, cd, bins), dtype=torch.uint8, device=DEV)
    ops.rvq_encode(xproj.to(DEV), 2 * cd, Ed, Et, en, codes, work, B * T, T, n_q, 1, cd, bins, time_major=True)
    torch.cuda.synchronize()
    ref = O.rvq_encode(z, w)
    margins = O.rvq_margins(z, w).min(dim=0).values.reshape(B, T)
    bad = (codes.cpu() != ref).any(dim=1)
    print(f"[codec-kernels] rvq time-major B={B} T={T}: {int(bad.sum())} of {B * T} frames differ, "
          f"all at margins <= 1e-4: {not bool((bad & (margins > 1e-4)).any())}")
    assert not bool((bad & (margins > 1e-4)).any())
    assert bad.float().mean().item() <= 0.05


def gather_ref(codes, E, ns, time_major):
    """q[n] = [sum_{l<ns} E_l[c_l] | sum_{l>=ns} E_l[c_l]] with fp32 adds in level order from +0."""
    B, n_q, T = codes.shape
    c = codes.clamp(0, E.shape[1] - 1)
    parts = [torch.zeros(B, T, E.shape[2]), torch.zeros(B, T, E.shape[2])]
    for l in range(n_q):
        gi = 0 if l < ns else 1
        parts[gi] = parts[gi] + E[l][c[:, l]]
    q = torch.cat(parts, -1)
    return q.transpose(0, 1).reshape(T * B, -1) if time_major else q.reshape(B * T, -1)


@pytest.mark.parametrize("time_major", [False, True])
def test_rvq_decode_gather_bit_exact(time_major, official_weights):
    B, n_q, T, bins, cd = 37, 8, 3, 2048, 256
    g = torch.Generator().manual_seed(2 + int(time_major))
    codes = torch.randint(0, bins, (B, n_q, T), generator=g)
    E, Ed, _, _ = _rvq_tables(official_weights)
    q = canvas(B * T * 2 * cd + 128)
    error_flags(True)
    ops.rvq_decode_gather(codes.to(DEV), Ed, q[64:], B * T, T, n_q, 1, cd, bins, time_major=time_major)
    torch.cuda.synchronize()
    got = q[64:64 + B * T * 2 * cd].view(B * T, 2 * cd).cpu()
    assert torch.equal(got, gather_ref(codes, E, 1, time_major))
    assert_canaries("rvq gather", q, torch.arange(64, 64 + B * T * 2 * cd, device=DEV))
    assert error_flags(True) == 0


def test_rvq_decode_gather_clamps_out_of_range(official_weights):
    """codes -1 and `bins` read the first / last centroid and set error bit 0 (F.embedding would raise)."""
    B, n_q, T, bins, cd = 4, 8, 2, 2048, 256
    codes = torch.randint(0, bins, (B, n_q, T), generator=torch.Generator().manual_seed(8))
    codes[1, 3, 0] = -1
    codes[2, 0, 1] = bins
    E, Ed, _, _ = _rvq_tables(official_weights)
    q = torch.empty(B * T, 2 * cd, device=DEV)
    error_flags(True)
    ops.rvq_decode_gather(codes.to(DEV), Ed, q, B * T, T, n_q, 1, cd, bins)
    torch.cuda.synchronize()
    assert error_flags(True) & 1
    assert torch.equal(q.cpu(), gather_ref(codes, E, 1, False))
    assert error_flags(True) == 0


# ============================================================================ small kernels
def fma_chain(pairs, init):
    acc, tie = init, torch.zeros(init.shape, dtype=torch.bool)
    for a, b in pairs:
        acc, t = fp32_fma(a, b, acc)
        tie |= t
    return acc, tie


@pytest.mark.parametrize("k,Cout,T,tm", [(1, 1, 100, False), (7, 32, 300, False), (16, 64, 257, True), (7, 200, 129, True)])
def test_conv1d_cin1(k, Cout, T, tm):
    """fmaf chain over the taps from +0, + bias, out and the ex2 ELU copy out2; time-major strides (tm)."""
    B = 3
    g = torch.Generator().manual_seed(k * Cout + T)
    x = torch.randn(B, T + k - 1, generator=g)
    w = torch.randn(Cout, k, generator=g)
    bias = torch.randn(Cout, generator=g)
    if tm:   # [T', B, 1] with samples B apart; out [T, B, Cout]
        xb = x.t().contiguous().to(DEV)
        x_bs, x_ts, o_bs, o_ts = 1, B, Cout, B * Cout
    else:
        xb = x.contiguous().to(DEV)
        x_bs, x_ts, o_bs, o_ts = T + k - 1, 1, T * Cout, Cout
    n = B * T * Cout
    out, out2 = canvas(n + 64), canvas(n + 64)
    ops.conv1d_cin1(xb, x_bs, x_ts, w.to(DEV), bias.to(DEV), out, 32, o_bs, o_ts, B, T, Cout, k, out2=out2, out2_off=32,
                    act2=ACT_ELU)
    torch.cuda.synchronize()
    win = x.unfold(1, k, 1)                                    # [B, T, k]
    acc, tie = fma_chain([(win[..., j:j + 1], w[:, j]) for j in range(k)], torch.zeros(B, T, Cout))
    ref = (acc.to(F64) + bias.to(F64)).to(F32)
    idx = strided_index(n + 64, (B, T, Cout), (o_bs, o_ts, 1), 32)
    exact_or_tie(f"conv1d_cin1 k={k} Cout={Cout}", out[idx].cpu(), ref, tie)
    check_bound(f"conv1d_cin1 out2 k={k} Cout={Cout}", out2[idx], act64(ref.to(F64).to(DEV), ACT_ELU), ELU_EX2)
    assert_canaries("conv1d_cin1", out, idx)
    assert_canaries("conv1d_cin1 out2", out2, idx)


@pytest.mark.parametrize("Cin,k,pad,off", [(64, 3, 0, 0), (32, 7, 0, 0), (64, 1, 0, 1), (16, 5, 2, 0), (6, 7, 0, 0),
                                           (6, 1, 0, 0), (100, 2, 0, 0)])
def test_conv1d_cout1(Cin, k, pad, off):
    """The three load paths: 16-byte (Cin % 4 == 0, aligned rows), power-of-two Cin with an unaligned row stride or base,
    any other Cin; the weight order is (tap, ci)."""
    B, T = 2, 200
    g = torch.Generator().manual_seed(Cin + k)
    rs = Cin + pad
    x = torch.randn(B, T + k - 1, rs, generator=g)
    w = torch.randn(k * Cin, generator=g) / math.sqrt(k * Cin)
    bias = torch.randn(1, generator=g)
    xflat = torch.cat([torch.zeros(off), x.reshape(-1)]).to(DEV)
    xv = xflat[off:] if off else xflat
    out = canvas(B * (T + 8) + 64)
    ops.conv1d_cout1(xv, (T + k - 1) * rs, rs, w.to(DEV), bias.to(DEV), out[16:], T + 8, B, T, Cin, k)
    torch.cuda.synchronize()
    pairs = [(x[:, j:j + T, c], w[j * Cin + c]) for j in range(k) for c in range(Cin)]
    acc, tie = fma_chain(pairs, torch.zeros(B, T))
    ref = (acc.to(F64) + bias.to(F64)).to(F32)   # one fp32 add
    idx = strided_index(B * (T + 8) + 64, (B, T), (T + 8, 1), 16)
    exact_or_tie(f"conv1d_cout1 Cin={Cin} k={k} pad={pad} off={off}", out[idx].cpu(), ref, tie)
    assert_canaries("conv1d_cout1", out, idx)


@pytest.mark.parametrize("s", [2, 5])
def test_convtr1d_depthwise(s):
    """out[b, t*s + j, c] = fmaf(x[t], w[c][j], x[t-1] * w[c][j+s]) (carry row in front)."""
    B, T, Cc = 3, 9, 68
    g = torch.Generator().manual_seed(s)
    x = torch.randn(B, T + 1, Cc, generator=g)
    w = torch.randn(Cc, 2 * s, generator=g)
    n = B * T * s * Cc
    out = canvas(n + 64)
    ops.convtr1d_depthwise(x.to(DEV), (T + 1) * Cc, Cc, w.to(DEV), out, 16, T * s * Cc, Cc, B, T, Cc, s)
    torch.cuda.synchronize()
    cur = x[:, 1:].unsqueeze(2)                     # [B, T, 1, C]
    prev = x[:, :-1].unsqueeze(2)
    wj, wjs = w[:, :s].t(), w[:, s:].t()            # [s, C]
    p = (prev.to(F64) * wjs.to(F64)).to(F32)        # fp32 product
    ref, tie = fp32_fma(cur, wj, p)
    idx = strided_index(n + 64, (B, T * s, Cc), (T * s * Cc, Cc, 1), 16)
    exact_or_tie(f"convtr1d_depthwise s={s}", out[idx].cpu(), ref.reshape(B, T * s, Cc), tie.reshape(B, T * s, Cc))
    assert_canaries("convtr1d_depthwise", out, idx)


@pytest.mark.parametrize("dim,rows", [(256, 7), (512, 13), (1024, 5), (384, 9), (96, 3)])
def test_layer_norm(dim, rows):
    """The register kernels (256 / 512 / 1024) and the generic one; row counts not a multiple of 4; mean >> std."""
    B = 3
    g = torch.Generator().manual_seed(dim + rows)
    x = torch.randn(B, rows + 2, dim, generator=g)
    x[1] += 1e3                                        # mean >> std
    w = torch.randn(dim, generator=g)
    b = torch.randn(dim, generator=g)
    y = canvas(B * rows * dim + 64)
    ops.layer_norm(x.to(DEV), dim, (rows + 2) * dim, w.to(DEV), b.to(DEV), y[32:], B, rows, dim, 1e-5)
    torch.cuda.synchronize()
    xs = x[:, 1:rows + 1].to(F64)
    mean, var = xs.mean(-1, keepdim=True), xs.var(-1, unbiased=False, keepdim=True)
    ref = (xs - mean) / torch.sqrt(var + 1e-5) * w.to(F64) + b.to(F64)
    slack = LN_C * (1 + mean.abs() / var.sqrt()) * w.to(F64).abs()
    check_bound(f"layer_norm dim={dim} rows={rows}", y[32:32 + B * rows * dim].view(B, rows, dim).cpu(), ref, slack)
    assert_canaries("layer_norm", y, torch.arange(32, 32 + B * rows * dim, device=DEV))


@pytest.mark.parametrize("layout", ["batch_major", "time_major"])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("oz", [None, "shared0", "shared1", "per_stream"])
def test_rows_fill(layout, mode, oz):
    S_, cps, rows = 5, 12, 9
    row0, nrows, src = 2, 3, 6
    g = torch.Generator().manual_seed(mode)
    if layout == "batch_major":
        batch, Cc, bs = S_, cps, rows * cps + 4
    else:
        batch, Cc, bs = 1, S_ * cps, 0
    n = (batch - 1) * bs + rows * Cc + 16
    buf = torch.randn(n, generator=g)
    counters = torch.tensor([0, 3, 0, 1, 0], dtype=torch.int64)
    ozt = {None: None, "shared0": torch.zeros(1, dtype=torch.int64), "shared1": torch.ones(1, dtype=torch.int64),
           "per_stream": counters}[oz]
    d = buf.to(DEV)
    ops.rows_fill(d, bs, batch, Cc, row0, nrows, mode=mode, src_row=src, only_if_zero=None if ozt is None else ozt.to(DEV),
                  channels_per_stream=cps)
    torch.cuda.synchronize()
    ref = buf.clone()
    for b in range(batch):
        for c in range(Cc):
            stream = b * (Cc // cps) + c // cps
            if ozt is not None and int(ozt[stream if ozt.numel() > 1 else 0]) != 0:
                continue
            for r in range(row0, row0 + nrows):
                ref[b * bs + r * Cc + c] = ref[b * bs + src * Cc + c] if mode == 1 else 0.0
    assert torch.equal(d.cpu().view(torch.int32), ref.view(torch.int32))


@pytest.mark.parametrize("layout", ["batch_major", "time_major"])
@pytest.mark.parametrize("held", [False, True])
def test_rows_copy_table(layout, held):
    """Overlapping carries (nrows > src - dst) move like memmove; a held stream keeps its rows; other bytes untouched."""
    S_, cps = 6, 20
    g = torch.Generator().manual_seed(int(held))
    active = torch.tensor([1, 0, 1, 1, 0, 1] if held else [1] * S_, dtype=torch.int64)
    ents = [(12, 0, 3, 20), (9, 1, 2, 10), (5, 0, 4, 20)]   # (rows, dst, src, cps): nrows = rows - src; the first two overlap
    bufs, entries = [], []
    for rows, dst, src, c in ents:
        if layout == "batch_major":
            batch, Cc, bs = S_, c, rows * c + 4
        else:
            batch, Cc, bs = 1, S_ * c, 0
        t = torch.randn((batch - 1) * bs + rows * Cc + 8, generator=g)
        bufs.append((t, batch, Cc, bs, rows, dst, src, c))
    dev = [b[0].to(DEV) for b in bufs]
    for (t, batch, Cc, bs, rows, dst, src, c), d in zip(bufs, dev):
        entries.append((d, bs, Cc, src, dst, rows - src, c))
    table = ops.make_copy_table(entries, DEV)
    nb = S_ if layout == "batch_major" else 1
    assert all(b[1] == nb for b in bufs)
    ops.rows_copy_table(table, len(entries), nb, active.to(DEV))
    torch.cuda.synchronize()
    for (t, batch, Cc, bs, rows, dst, src, c), d in zip(bufs, dev):
        ref = t.clone()
        nr = rows - src
        for b in range(batch):
            for col in range(Cc):
                if int(active[b * (Cc // c) + col // c]) == 0:
                    continue
                vals = [t[b * bs + (src + r) * Cc + col].item() for r in range(nr)]
                for r in range(nr):
                    ref[b * bs + (dst + r) * Cc + col] = vals[r]
        assert torch.equal(d.cpu().view(torch.int32), ref.view(torch.int32)), (layout, held, rows, dst, src)


@pytest.mark.parametrize("n", [1, 5, 300])
def test_counter_add(n):
    c0 = torch.arange(n, dtype=torch.int64) * 7 - 3
    active = (torch.arange(n) % 3 != 1).to(torch.int64)
    c = c0.to(DEV)
    ops.counter_add(c, 5, active.to(DEV))
    ops.counter_add(c, -2)
    torch.cuda.synchronize()
    assert torch.equal(c.cpu(), c0 + 5 * active - 2)


# ============================================================================ whole codec: one NaN sample
@pytest.mark.parametrize("tensor_cores", [False, True])
def test_codec_nan_sample_stays_in_its_stream(tensor_cores, official_weights):
    """One NaN in one stream of a B = 4 streaming run: the other streams' codes and PCM are bit-identical to a run
    without it, and the NaN stream's latent frames that the FFMA path makes non-finite are non-finite on this path too."""
    B, frames = 4, 2
    from specs import mimi_spec as S
    x = S.synthetic_audio(B, 1920 * frames, seed=5)
    xn = x.clone()
    xn[1, 0, 700] = float("nan")

    def run(audio, tc):
        m = codec.MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
        m.load_state_dict(official_weights, strict=True)
        m = m.to(DEV).eval()
        m.streaming_tensor_cores = tc
        codes, wavs, lats = [], [], []
        with torch.no_grad(), m.streaming(B):
            for i in range(frames):
                c = m.encode(audio[..., i * 1920:(i + 1) * 1920].to(DEV))
                plan = next(iter(m._stream_state.enc.values()))
                lat = plan.lat.view(-1, B, plan.lat.shape[-1]) if tc else plan.lat.view(B, -1, plan.lat.shape[-1]).transpose(0, 1)
                lats.append(lat.clone())
                codes.append(c)
                wavs.append(m.decode(c.clamp(0, 2047)))
        torch.cuda.synchronize()
        return torch.cat(codes, -1).cpu(), torch.cat(wavs, -1).cpu(), torch.cat(lats, 0).cpu()

    error_flags(True)
    c_ref, w_ref, _ = run(x, tensor_cores)
    c_nan, w_nan, lat_nan = run(xn, tensor_cores)
    _, _, lat_ffma = run(xn, False) if tensor_cores else (None, None, lat_nan)
    error_flags(True)
    others = [0, 2, 3]
    assert torch.equal(c_ref[others], c_nan[others])
    assert torch.equal(w_ref[others].view(torch.int32), w_nan[others].view(torch.int32))
    bad_ffma = ~torch.isfinite(lat_ffma[:, 1]).all(-1)     # [frames]
    assert bool(bad_ffma.any()), "the FFMA path absorbed the NaN"
    bad = ~torch.isfinite(lat_nan[:, 1]).all(-1)
    assert bool(bad[bad_ffma].all()), f"latent frames {bad_ffma.nonzero().flatten().tolist()} non-finite on the FFMA path, " \
                                      f"{bad.nonzero().flatten().tolist()} here"
