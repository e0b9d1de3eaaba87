"""Thin tensor-level wrappers over the C ABI (include/rstnet_b200.h).

PyTorch is plumbing here: it owns device memory and streams; all arithmetic happens in
librstnet_b200.so.  Every wrapper takes CUDA tensors, passes raw pointers + the current stream,
and raises on failure (no fallback path).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import ACT_ELU, ACT_GELU, ACT_NONE, GemmRowsArgs, RowCopy, TcGemmDesc  # noqa: F401


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.RstnetError("rstnet_b200 ops need CUDA tensors (there is no CPU path)")


def gemm_rows(A: torch.Tensor, a_off: int, a_bs: int, a_rs: int, Wt: torch.Tensor, C_: torch.Tensor, c_off: int,
              c_bs: int, c_rs: int, batch: int, rows: int, *, bias=None, scale=None, R=None, r_off: int = 0,
              r_bs: int = 0, r_rs: int = 0, pre_act: int = ACT_NONE, post_act: int = ACT_NONE, taps: int = 1,
              tap_stride: int = 0) -> None:
    """C[b,t,:] = post(R + scale*(pre(A_row(b,t)) @ Wt + bias)); offsets/strides in elements."""
    _cuda(A, Wt, C_, bias, scale, R)
    K, N = Wt.shape
    a = GemmRowsArgs()
    a.A = A.data_ptr() + 4 * a_off
    a.a_batch_stride, a.a_row_stride = a_bs, a_rs
    a.Wt = Wt.data_ptr()
    a.bias, a.scale = _p(bias), _p(scale)
    a.R = None if R is None else R.data_ptr() + 4 * r_off
    a.r_batch_stride, a.r_row_stride = r_bs, r_rs
    a.C = C_.data_ptr() + 4 * c_off
    a.c_batch_stride, a.c_row_stride = c_bs, c_rs
    a.batch, a.rows, a.N, a.K = batch, rows, N, K
    a.pre_act, a.post_act = pre_act, post_act
    a.taps, a.tap_stride = taps, tap_stride
    _lib.check(_lib.lib().rstnet_gemm_rows_f32(C.byref(a), _stream()), "gemm_rows_f32")


def tf32_split(w: torch.Tensor):
    """(hi, lo) with hi = tf32_rna(w), lo = tf32_rna(w - hi): one-time weight preparation for 3xTF32."""
    _cuda(w)
    w = w.contiguous()
    both = torch.empty((2,) + tuple(w.shape), dtype=w.dtype, device=w.device)   # hi and lo adjacent: one 3-D TMA box fetches both
    hi, lo = both[0], both[1]
    _lib.check(_lib.lib().rstnet_tf32_split_f32(w.data_ptr(), hi.data_ptr(), lo.data_ptr(), w.numel(), _stream()), "tf32_split")
    return hi, lo


class TcGemm:
    """A tensor-core (wgmma) GEMM plan bound to fixed buffers (rstnet_tc_gemm_create / run / destroy).

    D[(i,o), n] = sum_tap sum_c A[c, i + tap*tap_di, o*o_mul + tap*tap_do] * W[n, tap*Kc + c];
    offsets / strides in elements; see include/rstnet_b200.h."""

    def __init__(self, A, a_off, a_i_stride, a_o_stride, a_c_extent, a_i_extent, a_o_extent, W, Kc, C_, c_off, c_i_stride,
                 c_o_stride, I_out, O_out, *, taps=1, tap_di=0, tap_do=0, o_mul=1, bias=None, scale=None, R=None, r_off=0,
                 r_i_stride=0, r_o_stride=0, n_split=0, c_split_stride=0, r_split_stride=0, pre_act=ACT_NONE,
                 post_act=ACT_NONE, precision=0, W_lo=None, C2=None, c2_off=0, act2=ACT_NONE):
        _cuda(A, W, C_, bias, scale, R, W_lo)
        N, Ktot = W.shape
        if precision == 0 and W_lo is None:
            W, W_lo = tf32_split(W)
        assert Ktot == taps * Kc, (Ktot, taps, Kc)
        d = TcGemmDesc()
        d.A = A.data_ptr() + 4 * a_off
        d.a_i_stride, d.a_o_stride = a_i_stride, a_o_stride
        d.a_c_extent, d.a_i_extent, d.a_o_extent = a_c_extent, a_i_extent, a_o_extent
        d.taps, d.tap_di, d.tap_do, d.o_mul = taps, tap_di, tap_do, o_mul
        d.W, d.W_lo, d.N, d.Kc, d.I_out, d.O_out = W.data_ptr(), _p(W_lo), N, Kc, I_out, O_out
        d.C = C_.data_ptr() + 4 * c_off
        d.c_i_stride, d.c_o_stride, d.c_split_stride = c_i_stride, c_o_stride, c_split_stride
        d.R = None if R is None else R.data_ptr() + 4 * r_off
        d.r_i_stride, d.r_o_stride, d.r_split_stride = r_i_stride, r_o_stride, r_split_stride
        d.bias, d.scale = _p(bias), _p(scale)
        d.n_split, d.pre_act, d.post_act, d.precision = n_split, pre_act, post_act, precision
        d.C2 = None if C2 is None else C2.data_ptr() + 4 * c2_off
        d.act2 = act2
        self._keep = (A, W, W_lo, C_, bias, scale, R, C2)  # the plan embeds raw pointers
        self.flops = 2.0 * I_out * O_out * N * Ktot  # algorithmic (one fp32-equivalent product per MAC)
        # algorithmic HBM bytes of the launch: every input element once, the weights once (hi and lo), the output(s) once
        in_rows = min(a_o_extent, O_out * o_mul + (taps - 1) * max(tap_do, 0))
        n_out = I_out * O_out * N
        self.bytes = 4.0 * (a_c_extent * a_i_extent * in_rows + (2 if W_lo is not None else 1) * N * Ktot
                            + n_out * (2 if C2 is not None else 1) + (n_out if R is not None else 0))
        self._h = C.c_void_p()
        _lib.check(_lib.lib().rstnet_tc_gemm_create(C.byref(d), C.byref(self._h)), "tc_gemm_create")

    def run(self):
        _lib.check(_lib.lib().rstnet_tc_gemm_run(self._h, _stream()), "tc_gemm_run")

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                _lib.lib().rstnet_tc_gemm_destroy(h)
            except Exception:
                pass
            self._h = None


def conv1d_cin1(x, x_bs, x_ts, w, bias, out, out_off, out_bs, out_ts, batch, T, Cout, k, post_act=ACT_NONE, out2=None,
                out2_off=0, act2=ACT_NONE):
    _cuda(x, w, out, out2)
    _lib.check(_lib.lib().rstnet_conv1d_cin1_f32(x.data_ptr(), x_bs, x_ts, w.data_ptr(), _p(bias), out.data_ptr() + 4 * out_off,
                                                 None if out2 is None else out2.data_ptr() + 4 * out2_off, out_bs, out_ts,
                                                 batch, T, Cout, k, post_act, act2, _stream()), "conv1d_cin1")


def conv1d_cout1(x, x_bs, x_ts, w, bias, out, out_bs, batch, T, Cin, k):
    _cuda(x, w, out)
    _lib.check(_lib.lib().rstnet_conv1d_cout1_f32(x.data_ptr(), x_bs, x_ts, w.data_ptr(), _p(bias), out.data_ptr(), out_bs,
                                                  batch, T, Cin, k, _stream()), "conv1d_cout1")


def convtr1d_depthwise(x, x_bs, x_ts, w, out, out_off, out_bs, out_ts, batch, T, Cch, stride):
    _cuda(x, w, out)
    _lib.check(_lib.lib().rstnet_convtr1d_depthwise_f32(x.data_ptr(), x_bs, x_ts, w.data_ptr(), out.data_ptr() + 4 * out_off,
                                                        out_bs, out_ts, batch, T, Cch, stride, _stream()), "convtr1d_depthwise")


def rows_fill(buf, bs, batch, Cch, row0, nrows, mode=0, src_row=0, only_if_zero=None, channels_per_stream=0):
    """only_if_zero: int64 counter(s); one element = shared, more = one per stream (see the header)."""
    _cuda(buf)
    oz_stride = 1 if (only_if_zero is not None and only_if_zero.numel() > 1) else 0
    _lib.check(_lib.lib().rstnet_rows_fill_f32(buf.data_ptr(), bs, batch, Cch, row0, nrows, mode, src_row,
                                               _p(only_if_zero), oz_stride, channels_per_stream, _stream()), "rows_fill")


def rows_copy_table(table_dev: torch.Tensor, n_entries: int, batch: int, active: Optional[torch.Tensor] = None):
    _lib.check(_lib.lib().rstnet_rows_copy_table_f32(table_dev.data_ptr(), n_entries, batch, _p(active), _stream()), "rows_copy_table")


def make_copy_table(entries, device) -> torch.Tensor:
    """entries: list of (tensor, batch_stride, C, src_row, dst_row, nrows, channels_per_stream) -> device uint8 tensor."""
    arr = (RowCopy * len(entries))()
    for i, (t, bs, c, s, d, n, cps) in enumerate(entries):
        if n > 0 and not (s >= d):
            raise _lib.RstnetError("carry copy must move rows towards the front (src_row >= dst_row)")
        arr[i].buf, arr[i].batch_stride, arr[i].C, arr[i].src_row, arr[i].dst_row, arr[i].nrows = t.data_ptr(), bs, c, s, d, n
        arr[i].cps = cps
    raw = bytes(arr)
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(device)


def counter_add(counter: torch.Tensor, delta: int, active: Optional[torch.Tensor] = None):
    """every element of the int64 counter tensor += delta (one shared counter or one per stream; elements whose
    `active` flag is 0 are held)"""
    if active is not None and active.numel() != counter.numel():
        active = None
    _lib.check(_lib.lib().rstnet_counter_add(counter.data_ptr(), delta, counter.numel(), _p(active), _stream()), "counter_add")


def _ostride(offset: torch.Tensor) -> int:
    return 1 if offset.numel() > 1 else 0


def layer_norm(x, x_off, x_bs, w, b, y, batch, rows, dim, eps):
    _cuda(x, w, b, y)
    _lib.check(_lib.lib().rstnet_layer_norm_f32(x.data_ptr() + 4 * x_off, x_bs, w.data_ptr(), b.data_ptr(), y.data_ptr(),
                                                batch, rows, dim, eps, _stream()), "layer_norm")


def rope_kv_append(qkv, q_bs, q_ts, kv, offset, freqs, batch, T, H, D, cap):
    _cuda(qkv, kv, offset, freqs)
    _lib.check(_lib.lib().rstnet_rope_kv_append_f32(qkv.data_ptr(), q_bs, q_ts, kv.data_ptr(), offset.data_ptr(), _ostride(offset),
                                                    freqs.data_ptr(), batch, T, H, D, cap, _stream()), "rope_kv_append")


def rope_ring_attention(qkv, q_bs, q_ts, kv, offset, freqs, out, o_bs, o_ts, batch, T, H, D, cap, context):
    """rope_kv_append + ring_attention in one launch (streaming steps of 2 tokens, head size 64)."""
    _cuda(qkv, kv, offset, freqs, out)
    _lib.check(_lib.lib().rstnet_rope_ring_attention_f32(qkv.data_ptr(), q_bs, q_ts, kv.data_ptr(), offset.data_ptr(), _ostride(offset),
                                                         freqs.data_ptr(), out.data_ptr(), o_bs, o_ts, batch, T, H, D, cap, context,
                                                         _stream()), "rope_ring_attention")


def ring_attention(qkv, q_bs, q_ts, kv, offset, out, o_bs, o_ts, batch, T, H, D, cap, context, linear):
    _cuda(qkv, kv, offset, out)
    _lib.check(_lib.lib().rstnet_ring_attention_f32(qkv.data_ptr(), q_bs, q_ts, kv.data_ptr(), offset.data_ptr(), _ostride(offset),
                                                    out.data_ptr(), o_bs, o_ts, batch, T, H, D, cap, context, int(linear),
                                                    _stream()), "ring_attention")


def rvq_encode_workspace(N, n_q, dim, bins) -> int:
    return int(_lib.lib().rstnet_rvq_encode_workspace(N, n_q, dim, bins))


def rvq_encode(x, ldx, E, Et, enorm, codes, work, N, T, n_q, ns, dim, bins, time_major=False):
    _cuda(x, E, Et, enorm, codes, work)
    _lib.check(_lib.lib().rstnet_rvq_encode_f32(x.data_ptr(), ldx, E.data_ptr(), Et.data_ptr(), enorm.data_ptr(),
                                                codes.data_ptr(), work.data_ptr(), N, T, n_q, ns, dim, bins, int(time_major),
                                                _stream()), "rvq_encode")


def rvq_decode_gather(codes, E, q, N, T, n_q, ns, dim, bins, time_major=False):
    _cuda(codes, E, q)
    _lib.check(_lib.lib().rstnet_rvq_decode_gather_f32(codes.data_ptr(), E.data_ptr(), q.data_ptr(), N, T, n_q, ns, dim,
                                                       bins, int(time_major), _stream()), "rvq_decode_gather")
