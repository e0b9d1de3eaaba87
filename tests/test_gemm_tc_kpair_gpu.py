"""The tensor-core GEMM's K-pair mode (64-row tiles, promotion chunks alternating between the two consumer warpgroups)
against its 128-row mode, bit for bit: each case builds both plans with rstnet_tc_gemm_create_ex on the same inputs and
output canvases and compares every element of the output buffers, canaries included.  The 128-row mode is the one
tests/test_codec_kernels_gpu.py holds to float64.  Also: which mode rstnet_tc_gemm_create picks."""
import ctypes as C
import zlib

import pytest
import torch

from rstnet_b200 import _lib, ops
from rstnet_b200._lib import ACT_ELU, ACT_GELU, ACT_NONE

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENT = 0x7FBADBAD   # canary: a NaN no kernel writes
NAN = 0x7FFFFFFF


def canvas(n):
    return torch.full((n,), SENT, dtype=torch.int32, device=DEV).view(torch.float32)


def put(t, flat, bits):
    t.view(torch.int32)[flat] = torch.tensor(bits, dtype=torch.int64).to(torch.int32).item()


class Pair:
    """Inputs, output canvases and one descriptor; run(kpair) builds the plan in that mode, runs it on fresh copies of
    the canvases and returns them."""

    def __init__(self, prec, seed, *, I_out, O_out, N, Kc, taps=1, tap_di=0, tap_do=0, o_mul=1, bias=False, scale=False,
                 R=None, n_split=0, pre=ACT_NONE, post=ACT_NONE, C2=False, act2=ACT_ELU, nan=False):
        g = torch.Generator(device=DEV).manual_seed(seed)
        a_i_extent = I_out + (taps - 1) * tap_di
        a_o_extent = (O_out - 1) * o_mul + 1 + (taps - 1) * tap_do
        a_i_stride, a_off = Kc + 4, 16
        a_o_stride = a_i_extent * a_i_stride + 8
        self.A = torch.randn(a_off + a_o_extent * a_o_stride + 16, generator=g, device=DEV)
        W = torch.randn(N, taps * Kc, generator=g, device=DEV) / (taps * Kc) ** 0.5
        if nan:   # a NaN activation (one column of outputs), a NaN weight (one output column)
            put(self.A, a_off + (a_o_extent - 1) * a_o_stride + (a_i_extent // 2) * a_i_stride + 5, NAN)
            W.view(torch.int32)[N // 3, taps * Kc - 7] = NAN
        self.W, self.W_lo = (ops.tf32_split(W) if prec == 0 else (W, None))
        J = N // n_split if n_split else 1
        ns = n_split or N
        c_i_stride = ns + 4
        c_split_stride = I_out * c_i_stride + 8 if n_split else 0
        c_o_stride = J * (I_out * c_i_stride + 8) + 4 if n_split else I_out * c_i_stride + 12
        c_off = 32
        nc = c_off + O_out * c_o_stride + 64
        self.C0 = canvas(nc)
        self.C20 = canvas(nc) if C2 else None
        self.bias = torch.randn(N, generator=g, device=DEV) if bias else None
        self.scale = torch.rand(N, generator=g, device=DEV) + 0.5 if scale else None
        self.R = None
        d = _lib.TcGemmDesc()
        d.a_i_stride, d.a_o_stride = a_i_stride, a_o_stride
        d.a_c_extent, d.a_i_extent, d.a_o_extent = Kc, a_i_extent, a_o_extent
        d.taps, d.tap_di, d.tap_do, d.o_mul = taps, tap_di, tap_do, o_mul
        d.A = self.A.data_ptr() + 4 * a_off
        d.W, d.W_lo = self.W.data_ptr(), None if self.W_lo is None else self.W_lo.data_ptr()
        d.N, d.Kc, d.I_out, d.O_out = N, Kc, I_out, O_out
        d.c_i_stride, d.c_o_stride, d.c_split_stride = c_i_stride, c_o_stride, c_split_stride
        d.bias = None if self.bias is None else self.bias.data_ptr()
        d.scale = None if self.scale is None else self.scale.data_ptr()
        d.n_split, d.pre_act, d.post_act, d.precision = n_split, pre, post, prec
        d.act2 = act2
        if R == "inplace":   # the epilogue reads the residual where it writes
            self.C0.copy_(torch.randn(nc, generator=g, device=DEV))
            self.r_inplace, self.r_off = True, c_off
            d.r_i_stride, d.r_o_stride, d.r_split_stride = c_i_stride, c_o_stride, c_split_stride
        elif R == "sep":
            self.r_inplace = False
            self.R = torch.randn(nc + 40, generator=g, device=DEV)
            d.R = self.R.data_ptr() + 4 * 40
            d.r_i_stride, d.r_o_stride, d.r_split_stride = c_i_stride, c_o_stride, c_split_stride
        else:
            self.r_inplace = False
        self.d, self.c_off = d, c_off
        self.n_written = I_out * O_out * N

    def plan(self, kpair, Cb, C2b):
        self.d.C = Cb.data_ptr() + 4 * self.c_off
        self.d.C2 = None if C2b is None else C2b.data_ptr() + 4 * self.c_off
        if self.r_inplace:
            self.d.R = self.d.C
        h = C.c_void_p()
        _lib.check(_lib.lib().rstnet_tc_gemm_create_ex(C.byref(self.d), kpair, C.byref(h)), "tc_gemm_create_ex")
        on = C.c_int32(-1)
        assert _lib.lib().rstnet_tc_gemm_kpair(h, C.byref(on)) == 0
        return h, on.value

    def run(self, kpair):
        Cb = self.C0.clone()
        C2b = None if self.C20 is None else self.C20.clone()
        h, on = self.plan(kpair, Cb, C2b)
        try:
            assert on == kpair
            _lib.check(_lib.lib().rstnet_tc_gemm_run(h, torch.cuda.current_stream().cuda_stream), "tc_gemm_run")
            torch.cuda.synchronize()
        finally:
            _lib.lib().rstnet_tc_gemm_destroy(h)
        return Cb, C2b

    def check(self, name):
        a, a2 = self.run(0)
        b, b2 = self.run(1)
        changed = int((a.view(torch.int32) != self.C0.view(torch.int32)).sum())
        assert changed >= self.n_written * 0.99, f"{name}: only {changed} of {self.n_written} outputs written"
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), \
            f"{name}: {int((a.view(torch.int32) != b.view(torch.int32)).sum())} elements of C differ"
        if a2 is not None:
            assert torch.equal(a2.view(torch.int32), b2.view(torch.int32)), f"{name}: C2 differs"
        return a


CASES = {
    # the few-tile, long-K launches of the streaming codec at 256 streams
    "tr_out_w": dict(I_out=512, O_out=1, N=512, Kc=512, R="sep"),
    "tr_w2": dict(I_out=512, O_out=1, N=512, Kc=2048, R="sep"),
    "enc_final_k3": dict(I_out=256, O_out=2, N=512, Kc=1024, taps=3, tap_do=1),
    "enc_down_k4s2": dict(I_out=256, O_out=1, N=512, Kc=512, taps=4, tap_do=1, o_mul=2),
    "q_in": dict(I_out=256, O_out=1, N=512, Kc=512),
    # chunk counts: 1, 2, 3, odd with a short last chunk, even with a short last chunk
    "k1": dict(I_out=200, O_out=1, N=64, Kc=128, bias=True),
    "k2": dict(I_out=200, O_out=1, N=64, Kc=256, post=ACT_ELU, bias=True),
    "k3": dict(I_out=200, O_out=1, N=96, Kc=384, post=ACT_GELU, scale=True),
    "k5_short": dict(I_out=130, O_out=1, N=64, Kc=608),      # 19 stages: chunks 4+4+4+4+3
    "k2_short": dict(I_out=130, O_out=1, N=32, Kc=160),      # 5 stages: chunks 4+1
    # conv forms: I_out not a multiple of 64, O_out > 1 with taps and o_mul, taps along i
    "conv_I100": dict(I_out=100, O_out=3, N=64, Kc=192, taps=2, tap_do=1, o_mul=2, bias=True),
    "conv_taps_di": dict(I_out=129, O_out=1, N=68, Kc=96, taps=3, tap_di=1),
    "conv_s8_k16": dict(I_out=130, O_out=3, N=32, Kc=32, taps=16, tap_do=1, o_mul=8),
    # epilogue features
    "bias_scale_R": dict(I_out=150, O_out=2, N=96, Kc=512, bias=True, scale=True, R="sep"),
    "R_inplace": dict(I_out=70, O_out=2, N=64, Kc=384, bias=True, scale=True, R="inplace"),
    "C2_elu": dict(I_out=150, O_out=2, N=64, Kc=256, bias=True, C2=True, act2=ACT_ELU),
    "C2_post_gelu": dict(I_out=90, O_out=1, N=128, Kc=640, bias=True, C2=True, post=ACT_GELU, act2=ACT_ELU),
    "nsplit_C2": dict(I_out=130, O_out=3, N=128, Kc=256, taps=2, tap_do=1, bias=True, n_split=32, C2=True),
    "nsplit_R_post": dict(I_out=64, O_out=2, N=256, Kc=384, n_split=64, R="sep", post=ACT_ELU, scale=True),
    # many tiles per persistent CTA: the queue's slots and phases carry across tiles (odd and even chunk counts)
    "tiles_per_sm_k3": dict(I_out=20000, O_out=1, N=64, Kc=384, bias=True),
    "tiles_per_sm_k4": dict(I_out=9000, O_out=1, N=128, Kc=512, R="sep"),
    # NaN in A and in W propagates the same way
    "nan": dict(I_out=130, O_out=2, N=64, Kc=512, taps=2, tap_di=1, bias=True, nan=True),
}


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("prec", [0, 1])
@pytest.mark.parametrize("pre", [ACT_NONE, ACT_ELU])
def test_kpair_bit_identical(name, prec, pre):
    spec = dict(CASES[name])
    case = Pair(prec, seed=zlib.crc32(name.encode()) % 1000 + 7 * prec + pre, pre=pre, **spec)
    out = case.check(f"{name} prec={prec} pre={pre}")
    if spec.get("nan"):
        assert bool(out.isnan().sum() > (out.view(torch.int32) == SENT).sum()), "no NaN output beyond the canaries"


def expected_kpair(I_out, O_out, N, K, n_sms):
    """rstnet_tc_gemm_create's rule, after its tile-width rule: K-pair when the 128-row tiles fit in one round of the
    SMs and K-pair takes strictly fewer rounds times serial K stages per tile."""
    bn = 64 if N >= 64 else 32
    mt = -(-I_out // 128) * O_out
    if bn == 64 and -(-mt * -(-N // 32) // n_sms) * 2 <= -(-mt * -(-N // 64) // n_sms) * 3:
        bn = 32
    nt = -(-N // bn)
    t128, t64 = mt * nt, -(-I_out // 64) * O_out * nt
    stages = K // 32
    return t128 <= n_sms and -(-t64 // n_sms) * (-(-stages // 8) * 4) < stages


def test_kpair_choice():
    n = torch.cuda.get_device_properties(0).multi_processor_count
    shapes = {   # (I_out, N, K): K-pair expected on a 132-SM H100
        (512, 512, 512): True, (512, 512, 2048): True, (256, 512, 2048): True, (256, 512, 512): True,
        (512, 1536, 512): False, (512, 2048, 512): False, (512, 1024, 3584): False,   # ties: qkv, w1, a 32-wide k7 conv
        (24576, 256, 128): False, (200, 64, 128): False, (128 * n, 64, 1024): False,
        (122880, 256, 256): False,   # past one round of 128-row tiles, although the rounds alone would pick K-pair
    }
    for (I, N, K), want in shapes.items():
        assert expected_kpair(I, 1, N, K, n) == want or n != 132, (I, N, K)
        A = torch.zeros(I * K + 64, device=DEV)
        W = torch.zeros(N, K, device=DEV)
        Cb = torch.zeros(I * N + 64, device=DEV)
        plan = ops.TcGemm(A, 0, K, I * K, K, I, 1, W, K, Cb, 0, N, I * N, I, 1, precision=1)
        on = C.c_int32(-1)
        assert _lib.lib().rstnet_tc_gemm_kpair(plan._h, C.byref(on)) == 0
        assert bool(on.value) == expected_kpair(I, 1, N, K, n), (I, N, K, on.value)
        gx, gy, bn = C.c_int32(), C.c_int32(), C.c_int32()
        assert _lib.lib().rstnet_tc_gemm_grid(plan._h, C.byref(gx), C.byref(gy), C.byref(bn)) == 0
        assert gx.value == -(-I // 128) and gy.value == -(-N // bn.value)   # 128-row M tiles whatever the mode
        del plan


def test_kpair_refused():
    A = torch.zeros(4096, device=DEV)
    W = torch.zeros(64, 64, device=DEV)
    Cb = torch.zeros(4096, device=DEV)
    d = _lib.TcGemmDesc()
    d.A, d.a_i_stride, d.a_o_stride, d.a_c_extent, d.a_i_extent, d.a_o_extent = A.data_ptr(), 64, 64 * 32, 64, 32, 1
    d.taps, d.o_mul = 1, 1
    d.W, d.N, d.Kc, d.I_out, d.O_out = W.data_ptr(), 64, 64, 32, 1
    d.C, d.c_i_stride, d.c_o_stride = Cb.data_ptr(), 64, 64 * 32
    d.precision = 1
    h = C.c_void_p()
    assert _lib.lib().rstnet_tc_gemm_create_ex(C.byref(d), 2, C.byref(h)) != 0 and not h.value
    assert "kpair must be" in _lib.lib().rstnet_last_error().decode()
