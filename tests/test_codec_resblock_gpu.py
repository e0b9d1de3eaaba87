"""The fused tensor-core SEANet residual block (rstnet_tc_resblock_*, ops.TcResblock) on the GPU (-m gpu).

* Bit for bit against the two rstnet_tc_gemm launches it replaces (k3 conv C -> C/2 with ELU before and after into a
  hidden buffer, then the 1x1 conv C/2 -> C with the skip and the ELU that follows the block): same operations in the
  same order, so any difference is a bug.
* Against a float64 evaluation of the block, with the bound style of test_codec_kernels_gpu.py:
  |out - ref64| <= 2 ulp_fp32(ref64) + slack, the hidden tensor's own bound carried through the 1x1 conv.
* Output canaries: the output sits in a larger buffer of sentinel NaNs with gaps between streams and time steps.
* Whole codec: MimiCodec.fused_resblock on and off give identical codes and waveforms (streaming with held rows and a
  per-stream reset, a 256-stream streaming pass, a non-streaming tensor-core batch).
"""
import math

import pytest
import torch

from oracle import mimi_spec as S
from rstnet_b200 import ops
from rstnet_b200._lib import ACT_ELU
from rstnet_b200.codec import MimiCodec

pytestmark = pytest.mark.gpu
DEV, F32, F64 = "cuda", torch.float32, torch.float64
C0 = 2.0 ** -17          # 3xTF32
ELU_EX2 = 2.0 ** -21     # ex2.approx ELU, absolute
SENT = 0x7FBADBAD        # canary: a NaN no kernel writes


def ulp32(x):
    x = x.to(F64)
    _, e = torch.frexp(x.abs())
    e = torch.where(x == 0, torch.full_like(e, -125), e.clamp(min=-125))
    return torch.pow(2.0, (e - 24).to(F64))


def elu64(v):
    return torch.where(v > 0, v, torch.expm1(v))


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


class Block:
    """One residual block of C channels over B streams and T output steps: raw input y [(T + 2), B, C] (time-major, 2
    causal context rows), weights, the fused plan and the two-GEMM plans writing into separate canvases."""

    def __init__(self, Cc, B, T, seed=0, nan_at=None):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.Cc, self.B, self.T = Cc, B, T
        H = Cc // 2
        self.y = torch.randn(T + 2, B, Cc, generator=g, device=DEV)
        if nan_at is not None:   # (row, stream, channel)
            self.y[nan_at] = float("nan")
        self.W1 = torch.randn(H, 3 * Cc, generator=g, device=DEV) / math.sqrt(3 * Cc)
        self.b1 = torch.randn(H, generator=g, device=DEV) * 0.1
        self.W2 = torch.randn(Cc, H, generator=g, device=DEV) / math.sqrt(H)
        self.b2 = torch.randn(Cc, generator=g, device=DEV) * 0.1
        w1h, w1l = ops.tf32_split(self.W1)
        w2h, w2l = ops.tf32_split(self.W2)
        # output rows with gaps: stream stride C + 4, time stride B (C + 4) + 8, 16 elements before
        self.oi, self.oo, self.off = Cc + 4, B * (Cc + 4) + 8, 16
        o_ = torch.arange(T, device=DEV).view(-1, 1, 1)
        i_ = torch.arange(B, device=DEV).view(1, -1, 1)
        c_ = torch.arange(Cc, device=DEV).view(1, 1, -1)
        self.idx = self.off + o_ * self.oo + i_ * self.oi + c_
        n = int(self.idx.max()) + 1 + 64
        self.out = torch.full((n,), SENT, dtype=torch.int32, device=DEV).view(F32)
        self.out2 = self.out.clone()
        self.fused = ops.TcResblock(self.y, 0, Cc, B * Cc, T + 2, B, T, w1h, w1l, self.b1, w2h, w2l, self.b2, self.out, self.off,
                                    self.oi, self.oo)
        self.h = torch.empty(T, B, H, device=DEV)
        self.k3 = ops.TcGemm(self.y, 0, Cc, B * Cc, Cc, B, T + 2, w1h, Cc, self.h, 0, H, B * H, B, T, taps=3, tap_do=1,
                             bias=self.b1, pre_act=ACT_ELU, post_act=ACT_ELU, precision=0, W_lo=w1l)
        self.k1 = ops.TcGemm(self.h, 0, H, B * H, H, B, T, w2h, H, self.out2, self.off, self.oi, self.oo, B, T, bias=self.b2,
                             R=self.y, r_off=2 * B * Cc, r_i_stride=Cc, r_o_stride=B * Cc, post_act=ACT_ELU, precision=0,
                             W_lo=w2l)

    def run_fused(self):
        self.fused.run()
        torch.cuda.synchronize()
        return self.out[self.idx]

    def run_two(self):
        self.k3.run()
        self.k1.run()
        torch.cuda.synchronize()
        return self.out2[self.idx]

    def reference(self):
        """float64 block and its per-element bound."""
        Cc, T = self.Cc, self.T
        y = self.y.to(F64)
        ya = elu64(y)
        W1, W2 = self.W1.to(F64), self.W2.to(F64)
        acc = self.b1.to(F64).expand(T, self.B, -1).clone()
        S1 = self.b1.to(F64).abs().expand(T, self.B, -1).clone()
        for tap in range(3):
            Wt = W1[:, tap * Cc:(tap + 1) * Cc]
            acc += ya[tap:tap + T] @ Wt.t()
            S1 += ya[tap:tap + T].abs() @ Wt.abs().t()
        h = elu64(acc)
        # hidden bound: 3xTF32 products + the ex2 ELU of the operand (through |W1|) and of the result, then its own rounding
        hs = C0 * S1 + ELU_EX2 * W1.abs().sum(1) + ELU_EX2 + 2 * ulp32(h)
        r = y[2:]
        v = r + self.b2.to(F64) + h @ W2.t()
        slack = C0 * (h.abs() @ W2.abs().t() + self.b2.to(F64).abs() + r.abs()) + hs @ W2.abs().t() + ELU_EX2
        return elu64(v), slack


def assert_canaries(buf, idx):
    keep = torch.ones(buf.numel(), dtype=torch.bool, device=DEV)
    keep[idx.reshape(-1)] = False
    assert bool((buf.view(torch.int32)[keep] == SENT).all()), "elements outside the output were written"


CASES = [(Cc, B, T) for Cc in (64, 128) for B, T in ((3, 9), (128, 6), (256, 5))]


@pytest.mark.parametrize("Cc,B,T", CASES)
def test_resblock_equals_two_gemms(Cc, B, T):
    blk = Block(Cc, B, T, seed=Cc + B + T)
    fused, two = blk.run_fused(), blk.run_two()
    assert same_bits(fused, two), f"{int((fused != two).sum())} of {fused.numel()} outputs differ from the two-launch form"
    assert_canaries(blk.out, blk.idx)


@pytest.mark.parametrize("Cc", [64, 128])
def test_resblock_many_tiles_per_cta(Cc):
    """More tiles than SMs, a partial last stream tile: the persistent ring wraps across tiles with the held stages."""
    blk = Block(Cc, 200, 180, seed=3 + Cc)
    fused, two = blk.run_fused(), blk.run_two()
    assert same_bits(fused, two)
    assert_canaries(blk.out, blk.idx)


@pytest.mark.parametrize("Cc,B,T", [(64, 3, 9), (64, 256, 5), (128, 130, 7)])
def test_resblock_float64_bound(Cc, B, T):
    blk = Block(Cc, B, T, seed=11 * Cc + B)
    out = blk.run_fused().to(F64)
    ref, slack = blk.reference()
    err = (out - ref).abs()
    bound = 2 * ulp32(ref) + slack
    used = float((err / bound).max())
    print(f"[resblock] C={Cc} B={B} T={T}: worst {used:.4f} of the bound")
    assert bool((err <= bound).all()), f"{int((~(err <= bound)).sum())} outputs outside the bound"


@pytest.mark.parametrize("Cc", [64, 128])
def test_resblock_nan_stays_in_its_stream(Cc):
    B, T, s, row = 130, 6, 129, 4
    blk = Block(Cc, B, T, seed=5, nan_at=(row, s, 7))
    fused, two = blk.run_fused(), blk.run_two()
    assert bool(((fused == two) | (fused.isnan() & two.isnan())).all())
    others = torch.ones(B, dtype=torch.bool, device=DEV)
    others[s] = False
    assert bool(torch.isfinite(fused[:, others]).all()), "a NaN leaked into another stream"
    # output steps that read row `row` (t = row - 2 .. row, the k3 taps) are NaN; the others stay finite
    hit = torch.zeros(T, dtype=torch.bool, device=DEV)
    hit[max(0, row - 2):row + 1] = True
    assert bool(fused[hit, s].isnan().any(-1).all()) and bool(torch.isfinite(fused[~hit, s]).all())
    assert_canaries(blk.out, blk.idx)


def _codec(w, fused):
    m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(w, strict=True)
    m = m.to(DEV).eval()
    m.fused_resblock = fused
    return m


def test_codec_streaming_held_rows_and_reset(official_weights):
    """Streaming over several steps with rows held (set_active) and one stream restarted: codes and PCM are the same
    with and without the fused blocks."""
    B = 4
    x = S.synthetic_audio(B, 1920 * 6, seed=91).to(DEV)
    res = []
    for fused in (True, False):
        m = _codec(official_weights, fused)
        cs, ws = [], []
        with torch.no_grad(), m.streaming(B):
            for i in range(6):
                if i == 2:
                    m.set_active_streams([1, 0, 1, 1])
                if i == 3:
                    m.set_active_streams(None)
                if i == 4:
                    m.reset_streaming([2])
                c = m.encode(x[..., i * 1920:(i + 1) * 1920])
                cs.append(c)
                ws.append(m.decode(c))
        res.append((torch.cat(cs, -1), torch.cat(ws, -1)))
    assert torch.equal(res[0][0], res[1][0])
    assert same_bits(res[0][1], res[1][1])


def test_codec_256_streams(official_weights):
    B = 256
    x = S.synthetic_audio(B, 1920 * 3, seed=17).to(DEV)
    res = []
    for fused in (True, False):
        m = _codec(official_weights, fused)
        cs, ws = [], []
        with torch.no_grad(), m.streaming(B):
            for i in range(3):
                c = m.encode(x[..., i * 1920:(i + 1) * 1920])
                cs.append(c)
                ws.append(m.decode(c))
        res.append((torch.cat(cs, -1), torch.cat(ws, -1)))
        del m
        torch.cuda.empty_cache()
    assert torch.equal(res[0][0], res[1][0])
    assert same_bits(res[0][1], res[1][1])


def test_codec_batch_tensor_cores(official_weights):
    """Non-streaming batches of at least batch_tensor_cores_min clips run the tensor-core plans: fused or not, the same."""
    B = 96
    x = S.synthetic_audio(B, 1920 * 2, seed=23).to(DEV)
    res = []
    for fused in (True, False):
        m = _codec(official_weights, fused)
        with torch.no_grad():
            c = m.encode(x)
            res.append((c, m.decode(c)))
        del m
        torch.cuda.empty_cache()
    assert torch.equal(res[0][0], res[1][0])
    assert same_bits(res[0][1], res[1][1])
