"""Sample-rate conversion on the GPU: `torchaudio.transforms.Resample(orig, new)` with its default arguments, the call the
reference makes wherever it reads audio (MLLM_v2/tools/tokenizer/MimiCodec/mimi_tokenizer.py:40,67;
MLLM_v2/egs/moshi_ft/data_scripts/offline_tokenization.py:51; AudioCodec/MimiCodec/inference.py:24-34).

  * `Resample(orig_freq, new_freq)` -- the transform: its sinc / Hann table is built once on the host in float64 with the
    same torch ops as torchaudio's `_get_sinc_resample_kernel` (transform form: `dtype=None`), rounded to fp32, trimmed to
    each phase's run of nonzero taps and uploaded; `forward` is one `rstnet_resample_f32` launch (batch form).
  * `StreamingResampler(orig_freq, new_freq, batch, device)` -- per-stream streaming with the same table for a batch of
    real-time sessions: each call takes `[B, chunk]` (chunk a whole number of `o`-sample blocks) and returns
    `[B, chunk / o * n]`, the output of `Resample` on the stream's input preceded by `delay_blocks * o` zeros -- a fixed
    delay of `latency_samples` output samples -- bit for bit equal to the batch form on that input.

There is no CPU path: input must be a CUDA fp32 tensor.  torchaudio is not needed at run time.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch

from . import _lib, ops
from ._lib import RstnetError

LOWPASS_FILTER_WIDTH = 6       # torchaudio.transforms.Resample defaults (sinc_interp_hann)
ROLLOFF = 0.99
CARRY_COPY_ROWS = 8            # samples per entry of the carry-shift copy table (entries run in parallel)


def _int_rate(f, name: str) -> int:
    if isinstance(f, bool) or not isinstance(f, (int, float)) or int(f) != f or int(f) <= 0:
        raise RstnetError(f"{name} must be a positive integer sample rate, got {f!r} (resampling needs integer rates)")
    return int(f)


@dataclass
class ResampleTable:
    """The trimmed polyphase table of Resample(orig_freq, new_freq): `taps` fp32 [n, S] (phase p's nonzero run, zero
    padded at the end), `start` int32 [n] (first tap of the run within the full [n, K] table), K = 2 * width + o."""
    orig_freq: int
    new_freq: int
    o: int
    n: int
    width: int
    K: int
    taps: torch.Tensor
    start: torch.Tensor

    @property
    def S(self) -> int:
        return int(self.taps.shape[1])

    @property
    def start_max(self) -> int:
        return int(self.start.max())

    def expand(self) -> torch.Tensor:
        """The full fp32 [n, K] table back from the trimmed one."""
        full = torch.zeros(self.n, self.K, dtype=torch.float32)
        for p in range(self.n):
            s = int(self.start[p])
            run = min(self.S, self.K - s)
            full[p, s:s + run] = self.taps[p, :run]
        return full


def reduced_rates(orig_freq, new_freq):
    """(o, n, width): input samples per block, output phases per block, and the table's half width."""
    orig, new = _int_rate(orig_freq, "orig_freq"), _int_rate(new_freq, "new_freq")
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    width = math.ceil(LOWPASS_FILTER_WIDTH * o / (min(o, n) * ROLLOFF))
    return o, n, width


def sinc_table(orig_freq, new_freq):
    """(fp32 [n, K] table, width): torchaudio.functional.functional._get_sinc_resample_kernel with the transform's
    defaults (sinc_interp_hann, width 6, rolloff 0.99, dtype None: built in float64, rounded to fp32)."""
    o, n, width = reduced_rates(orig_freq, new_freq)
    base_freq = min(o, n) * ROLLOFF
    idx = torch.arange(-width, width + o, dtype=torch.float64)[None, None] / o
    t = torch.arange(0, -n, -1, dtype=torch.float32)[:, None, None] / n + idx
    t *= base_freq
    t = t.clamp_(-LOWPASS_FILTER_WIDTH, LOWPASS_FILTER_WIDTH)
    window = torch.cos(t * math.pi / LOWPASS_FILTER_WIDTH / 2) ** 2
    t *= math.pi
    scale = base_freq / o
    kernels = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    kernels *= window * scale
    return kernels.to(torch.float32)[:, 0], width


def table_bytes_bound(orig_freq, new_freq) -> int:
    """Upper bound of the trimmed table's size, from the rates alone: a tap is nonzero only where the clamped sinc
    argument is inside (-6, 6), at most 2 * width + 1 consecutive taps of a phase."""
    o, n, width = reduced_rates(orig_freq, new_freq)
    return 4 * n * min(2 * width + o, 2 * width + 1)


def resample_table(orig_freq, new_freq) -> ResampleTable:
    """Build, round and trim the table (host, one time).  Refuses rates whose trimmed table would exceed the kernel's
    cap before building anything."""
    o, n, width = reduced_rates(orig_freq, new_freq)
    if table_bytes_bound(orig_freq, new_freq) > _lib.RESAMPLE_MAX_TABLE_BYTES:
        raise RstnetError(
            f"resampling {orig_freq} Hz -> {new_freq} Hz needs {n} filter phases of up to {2 * width + 1} taps "
            f"(about {table_bytes_bound(orig_freq, new_freq)} bytes), above the {_lib.RESAMPLE_MAX_TABLE_BYTES}-byte cap "
            "of the resampling kernel; pick rates with a larger common divisor")
    full, width = sinc_table(orig_freq, new_freq)
    K = full.shape[1]
    nz = full != 0
    any_nz = nz.any(dim=1)
    cols = torch.arange(K)
    first = torch.where(nz, cols, K).min(dim=1).values
    last = torch.where(nz, cols, -1).max(dim=1).values
    start = torch.where(any_nz, first, 0)
    length = torch.where(any_nz, last + 1 - first, 0)
    S = max(1, int(length.max()))
    taps = torch.zeros(n, S, dtype=torch.float32)
    for p in range(n):
        taps[p, :int(length[p])] = full[p, int(start[p]):int(start[p]) + int(length[p])]
    if 4 * n * S > _lib.RESAMPLE_MAX_TABLE_BYTES:
        raise RstnetError(f"resampling {orig_freq} Hz -> {new_freq} Hz: trimmed table {n} x {S} exceeds the "
                          f"{_lib.RESAMPLE_MAX_TABLE_BYTES}-byte cap")
    return ResampleTable(int(orig_freq), int(new_freq), o, n, width, K, taps, start.to(torch.int32))


def _check_input(x, what: str) -> None:
    if not isinstance(x, torch.Tensor):
        raise RstnetError(f"{what}: expected a torch.Tensor, got {type(x).__name__}")
    if not x.is_cuda:
        raise RstnetError(f"{what}: input must be a CUDA tensor (there is no CPU path)")
    if x.dtype != torch.float32:
        raise RstnetError(f"{what}: input must be float32, got {x.dtype}")


class _DeviceTable:
    def __init__(self, table: ResampleTable):
        self.table = table
        self._dev: Dict[torch.device, tuple] = {}

    def on(self, device):
        device = torch.device(device)
        if device not in self._dev:
            self._dev[device] = (self.table.taps.to(device), self.table.start.to(device))
        return self._dev[device]

    def launch(self, x, x_row_stride, x_len, x_shift, out, out_row_stride, out_len, rows):
        t = self.table
        taps, start = self.on(x.device)
        _lib.check(_lib.lib().rstnet_resample_f32(x.data_ptr(), x_row_stride, x_len, x_shift, taps.data_ptr(), start.data_ptr(),
                                                  t.n, t.o, t.S, t.start_max, out.data_ptr(), out_row_stride, out_len, rows,
                                                  ops._stream()), "resample")


class Resample:
    """torchaudio.transforms.Resample(orig_freq, new_freq) (default arguments) on the GPU: `forward` takes a CUDA fp32
    tensor [..., L] and returns [..., ceil(n * L / o)] in one launch; orig_freq == new_freq returns the input itself."""

    def __init__(self, orig_freq: int = 16000, new_freq: int = 16000):
        self.orig_freq, self.new_freq = _int_rate(orig_freq, "orig_freq"), _int_rate(new_freq, "new_freq")
        self._t: Optional[_DeviceTable] = None
        if self.orig_freq != self.new_freq:
            self._t = _DeviceTable(resample_table(self.orig_freq, self.new_freq))

    @property
    def table(self) -> Optional[ResampleTable]:
        return None if self._t is None else self._t.table

    def output_length(self, L: int) -> int:
        if self._t is None:
            return L
        t = self._t.table
        return int(math.ceil(t.n * L / t.o))            # torch.ceil(new_freq * length / orig_freq), as torchaudio

    def forward(self, waveform: torch.Tensor) -> torch.Tensor:
        _check_input(waveform, "Resample")
        if self._t is None:
            return waveform
        shape = waveform.shape
        L = shape[-1]
        x = waveform.reshape(-1, L)
        if L > 1 and x.stride(1) != 1:
            x = x.contiguous()
        rows, out_len = x.shape[0], self.output_length(L)
        out = torch.empty(rows, out_len, dtype=torch.float32, device=x.device)
        if rows and out_len:
            self._t.launch(x, x.stride(0), L, -self._t.table.width, out, out_len, out_len, rows)
        return out.view(shape[:-1] + (out_len,))

    __call__ = forward


class StreamingResampler:
    """Per-stream streaming Resample(orig_freq, new_freq) for `batch` rows.  Every call takes [batch, chunk] (chunk a
    multiple of o) and returns [batch, chunk / o * n]: the continuation of Resample applied to each stream's input
    preceded by delay_blocks * o zeros.  A row keeps a carry of delay_blocks * o + width input samples; `reset(rows)`
    restarts rows, `set_active(mask)` holds rows whose flag is 0 (their carry does not advance)."""

    def __init__(self, orig_freq: int, new_freq: int, batch: int, device):
        self.orig_freq, self.new_freq = _int_rate(orig_freq, "orig_freq"), _int_rate(new_freq, "new_freq")
        if self.orig_freq == self.new_freq:
            raise RstnetError("StreamingResampler: orig_freq == new_freq, there is nothing to resample")
        if batch < 1:
            raise RstnetError(f"StreamingResampler: batch must be >= 1, got {batch}")
        self.B, self.device = int(batch), torch.device(device)
        self._t = _DeviceTable(resample_table(self.orig_freq, self.new_freq))
        t = self._t.table
        self.o, self.n, self.width = t.o, t.n, t.width
        self.delay_blocks = -(-t.width // t.o)                 # D = ceil(width / o)
        self.carry = self.delay_blocks * t.o + t.width
        self.latency_samples = self.delay_blocks * t.n          # output samples of delay
        self.active = torch.ones(self.B, dtype=torch.int64, device=self.device)
        self._buf: Optional[torch.Tensor] = None
        self._chunk = 0
        self._copy_table: Optional[torch.Tensor] = None
        self._copy_entries = 0

    def output_length(self, chunk: int) -> int:
        if chunk % self.o:
            raise RstnetError(f"StreamingResampler {self.orig_freq} -> {self.new_freq} Hz: a chunk must be a multiple of "
                              f"{self.o} samples, got {chunk}")
        return chunk // self.o * self.n

    def _ensure(self, chunk: int) -> None:
        if chunk == self._chunk:
            return
        buf = torch.zeros(self.B, self.carry + chunk, dtype=torch.float32, device=self.device)
        if self._buf is not None:
            buf[:, :self.carry].copy_(self._buf[:, :self.carry])
        self._buf, self._chunk = buf, chunk
        # carry shift: buf[:, 0:carry] = buf[:, chunk:chunk + carry], rows_copy_table over [B, carry + chunk, C = 1];
        # when source and destination do not overlap the copy is split into entries that run in parallel
        bs = self.carry + chunk
        if chunk >= self.carry:
            entries = [(buf, bs, 1, chunk + k, k, min(CARRY_COPY_ROWS, self.carry - k), 1)
                       for k in range(0, self.carry, CARRY_COPY_ROWS)]
        else:
            entries = [(buf, bs, 1, chunk, 0, self.carry, 1)]
        self._copy_table, self._copy_entries = ops.make_copy_table(entries, self.device), len(entries)

    def __call__(self, x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        _check_input(x, "StreamingResampler")
        if x.dim() != 2 or x.shape[0] != self.B:
            raise RstnetError(f"StreamingResampler: expected [{self.B}, chunk], got {tuple(x.shape)}")
        chunk = x.shape[1]
        out_len = self.output_length(chunk)
        if out is None:
            out = torch.empty(self.B, out_len, dtype=torch.float32, device=self.device)
        elif out.shape != (self.B, out_len) or out.dtype != torch.float32 or out.device != self.device or out.stride(1) != 1:
            raise RstnetError(f"StreamingResampler: `out` must be a float32 [{self.B}, {out_len}] tensor with contiguous rows on {self.device}")
        if chunk == 0:
            return out
        self._ensure(chunk)
        self._buf[:, self.carry:].copy_(x)
        bs = self.carry + chunk
        self._t.launch(self._buf, bs, bs, 0, out, out.stride(0), out_len, self.B)
        ops.rows_copy_table(self._copy_table, self._copy_entries, self.B, self.active)
        return out

    def row_segments(self, b: int, chunk: int):
        """Row b's state as row_state regions: its carry of `carry` input samples (the buffer for `chunk`-sample calls is
        built here if no call has built it yet)."""
        from .row_state import segs
        self._ensure(chunk)
        n = self.carry * self._buf.element_size()
        return [("carry", segs((self._buf[b].data_ptr(), n, n, 1)))]

    def reset(self, rows=None) -> None:
        """Zero the carry of `rows` (None = all): those streams restart as fresh streams."""
        if self._buf is None:
            return
        bs = self.carry + self._chunk
        if rows is None:
            ops.rows_fill(self._buf, bs, self.B, 1, 0, self.carry)
            return
        for r in rows:
            r = int(r)
            if not 0 <= r < self.B:
                raise RstnetError(f"stream index {r} outside [0, {self.B})")
            ops.rows_fill(self._buf[r], bs, 1, 1, 0, self.carry)

    def set_active(self, mask) -> None:
        """mask [B]: rows whose flag is 0 are held by the following calls (their output is not meaningful and their
        carry does not advance).  None = every row advances."""
        if mask is None:
            self.active.fill_(1)
        else:
            self.active.copy_(torch.as_tensor(mask).to(device=self.device, dtype=torch.int64).reshape(self.B))
