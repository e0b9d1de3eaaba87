"""Tensor-core wgmma GEMM (rstnet_tc_gemm_*) vs the CPU oracle: linear, strided causal conv and transposed
conv in the time-major/batch-inner layout used by the streaming plans.  Precision 0 (3xTF32) must
be fp32-equivalent (<= 3e-6 relative to the fp32 result scale); precision 1 (TF32) ~1e-3."""
import pytest
import torch
import torch.nn.functional as F

from oracle import mimi_oracle as O
from rstnet_b200 import ops
from rstnet_b200._lib import ACT_ELU, ACT_GELU, ACT_NONE

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp(min=1e-6)).item()


@pytest.mark.parametrize("M,K,N", [(128, 32, 32), (256, 512, 512), (512, 2048, 512), (200, 512, 1536), (64, 64, 128), (300, 96, 36),
                                   (38400, 96, 64), (40000, 32, 64), (25000, 256, 128)])  # several tiles per persistent CTA, padded K loops
@pytest.mark.parametrize("prec,tol", [(0, 2e-6), (1, 3e-3)])
def test_tc_linear(M, K, N, prec, tol):
    g = torch.Generator().manual_seed(M + K + N)
    a = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = (a.double() @ w.double().t() + b.double()).float()
    ad, wd, out = a.to(DEV), w.to(DEV).contiguous(), torch.full((M, N), 7.0, device=DEV)
    plan = ops.TcGemm(ad, 0, K, M * K, K, M, 1, wd, K, out, 0, N, M * N, M, 1, bias=b.to(DEV), precision=prec)
    plan.run()
    torch.cuda.synchronize()
    err = _rel(out, ref)
    print(f"tc_linear M={M} K={K} N={N} prec={prec}: rel err {err:.2e}")
    assert err <= tol


def test_tc_linear_epilogues_inplace():
    g = torch.Generator().manual_seed(3)
    M, K, N = 384, 512, 2048
    a = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    ref = F.gelu(F.linear(a.double(), w.double())).float()
    ad, out = a.to(DEV), torch.empty(M, N, device=DEV)
    ops.TcGemm(ad, 0, K, M * K, K, M, 1, w.to(DEV), K, out, 0, N, M * N, M, 1, post_act=ACT_GELU).run()
    assert _rel(out, ref) <= 3e-6
    x = torch.randn(M, K, generator=g)
    w2 = torch.randn(K, N, generator=g) / N ** 0.5
    sc = torch.rand(K, generator=g)
    ref2 = (x.double() + sc.double() * F.linear(ref.double(), w2.double())).float()
    xd = x.to(DEV).clone()
    ops.TcGemm(out, 0, N, M * N, N, M, 1, w2.to(DEV), N, xd, 0, K, M * K, M, 1, scale=sc.to(DEV), R=xd, r_i_stride=K, r_o_stride=M * K).run()
    torch.cuda.synchronize()
    assert _rel(xd, ref2) <= 5e-6


@pytest.mark.parametrize("B,Cin,Cout,k,s,T", [(256, 64, 32, 3, 1, 6), (256, 64, 128, 8, 4, 8), (128, 128, 256, 10, 5, 10),
                                             (256, 512, 1024, 16, 8, 16), (256, 1024, 512, 3, 1, 2), (96, 256, 512, 12, 6, 12)])
@pytest.mark.parametrize("pre,post", [(ACT_NONE, ACT_NONE), (ACT_ELU, ACT_ELU)])
def test_tc_conv_time_major(B, Cin, Cout, k, s, T, pre, post):
    """causal strided conv over a [ctx+T, B, Cin] buffer: taps loop, o_mul = stride."""
    g = torch.Generator().manual_seed(Cin + k + B)
    x = torch.randn(B, Cin, T, generator=g)
    w = torch.randn(Cout, Cin, k, generator=g) / (Cin * k) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    xin = F.elu(x) if pre else x
    ref = O.causal_conv1d(xin.double(), w.double(), b.double(), stride=s)
    if post:
        ref = F.elu(ref)
    Tout = ref.shape[-1]
    ctx = k - s
    assert T % s == 0
    buf = torch.zeros(ctx + T, B, Cin, device=DEV)
    buf[ctx:] = x.permute(2, 0, 1).to(DEV)
    W = w.permute(0, 2, 1).reshape(Cout, k * Cin).contiguous().to(DEV)     # [N][(tap, ci)]
    out = torch.empty(Tout, B, Cout, device=DEV)
    plan = ops.TcGemm(buf, 0, Cin, B * Cin, Cin, B, ctx + T, W, Cin, out, 0, Cout, B * Cout, B, Tout, taps=k, tap_do=1,
                      o_mul=s, bias=b.to(DEV), pre_act=pre, post_act=post)
    plan.run()
    torch.cuda.synchronize()
    err = _rel(out.permute(1, 2, 0), ref.float())
    print(f'conv err {err:.2e}')
    assert err <= 2e-6


@pytest.mark.parametrize("B,Cin,Cout,s,T", [(256, 1024, 512, 8, 2), (256, 128, 64, 4, 10), (64, 256, 128, 5, 7)])
def test_tc_convtr_time_major(B, Cin, Cout, s, T):
    """ConvTranspose1d k=2s as a 2-tap GEMM over [x[t-1], x[t]] with the column-split epilogue."""
    g = torch.Generator().manual_seed(Cin + s)
    x = torch.randn(B, Cin, T, generator=g)
    w = torch.randn(Cin, Cout, 2 * s, generator=g) / (2 * Cin) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    ref = O.causal_convtr1d(x.double(), w.double(), b.double(), stride=s).float()
    buf = torch.zeros(1 + T, B, Cin, device=DEV)
    buf[1:] = x.permute(2, 0, 1).to(DEV)
    # W[n=(j,co)][(half,ci)]: half 0 = x[t-1] with tap j+s, half 1 = x[t] with tap j
    w_prev = w[:, :, s:].permute(2, 1, 0).reshape(s * Cout, Cin)
    w_cur = w[:, :, :s].permute(2, 1, 0).reshape(s * Cout, Cin)
    W = torch.cat([w_prev, w_cur], 1).contiguous().to(DEV)
    out = torch.empty(T * s, B, Cout, device=DEV)
    plan = ops.TcGemm(buf, 0, Cin, B * Cin, Cin, B, 1 + T, W, Cin, out, 0, Cout, s * B * Cout, B, T, taps=2, tap_do=1,
                      bias=b.repeat(s).to(DEV), n_split=Cout, c_split_stride=B * Cout)
    plan.run()
    torch.cuda.synchronize()
    err = _rel(out.permute(1, 2, 0), ref)
    print(f'convtr err {err:.2e}')
    assert err <= 2e-6
