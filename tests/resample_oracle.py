"""CPU restatement of torchaudio.transforms.Resample(orig, new) with its default arguments, in torch ops (test
infrastructure only; the product never imports torchaudio or this module).

Restates torchaudio 2.11's `torchaudio.functional.functional._get_sinc_resample_kernel` (sinc_interp_hann,
lowpass_filter_width 6, rolloff 0.99, dtype None: built in float64, rounded to fp32) and `_apply_sinc_resample_kernel`
(pad w zeros left and w + o right, conv1d with stride o, truncate to ceil(n * L / o)), plus the streaming definition of
rstnet_b200.audio.StreamingResampler: the batch transform of the stream's input preceded by D * o zeros (D = ceil(w/o)),
truncated to the samples the chunks seen so far determine.
"""
from __future__ import annotations

import hashlib
import math

import torch

# the pairs the project resamples between (client rates <-> the codec's 24 kHz)
PAIRS = [(16000, 24000), (44100, 24000), (48000, 24000), (8000, 24000), (22050, 24000), (11025, 24000),
         (24000, 16000), (24000, 48000), (24000, 8000)]
TORCHAUDIO_VERSION = "2.11.0"


def reduced(orig: int, new: int):
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    width = math.ceil(6 * o / (min(o, n) * 0.99))
    return o, n, width


def sinc_kernel(orig: int, new: int):
    """(fp32 [n, 1, K] conv1d weight, width), as _get_sinc_resample_kernel(orig, new, gcd) with dtype None."""
    o, n, width = reduced(orig, new)
    base_freq = min(o, n) * 0.99
    idx = torch.arange(-width, width + o, dtype=torch.float64)[None, None] / o
    t = torch.arange(0, -n, -1)[:, None, None] / n + idx      # int64 / int -> default float dtype, then float64
    t *= base_freq
    t = t.clamp_(-6, 6)
    window = torch.cos(t * math.pi / 6 / 2) ** 2
    t *= math.pi
    scale = base_freq / o
    kernels = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    kernels *= window * scale
    return kernels.to(dtype=torch.float32), width


def apply_kernel(waveform: torch.Tensor, orig: int, new: int, kernel: torch.Tensor, width: int) -> torch.Tensor:
    o, n, _ = reduced(orig, new)
    shape = waveform.size()
    waveform = waveform.view(-1, shape[-1])
    num_wavs, length = waveform.shape
    waveform = torch.nn.functional.pad(waveform, (width, width + o))
    resampled = torch.nn.functional.conv1d(waveform[:, None], kernel, stride=o)
    resampled = resampled.transpose(1, 2).reshape(num_wavs, -1)
    target_length = torch.ceil(torch.as_tensor(n * length / o)).long()
    resampled = resampled[..., :target_length]
    return resampled.view(shape[:-1] + resampled.shape[-1:])


def resample(waveform: torch.Tensor, orig: int, new: int) -> torch.Tensor:
    if orig == new:
        return waveform
    kernel, width = sinc_kernel(orig, new)
    return apply_kernel(waveform, orig, new, kernel, width)


def trim(table: torch.Tensor):
    """fp32 [n, K] -> (taps [n, S] zero-padded runs, start int32 [n]); asserts the table is zero outside the runs."""
    n, K = table.shape
    starts, runs = [], []
    for p in range(n):
        nz = torch.nonzero(table[p]).flatten()
        s, e = (int(nz[0]), int(nz[-1]) + 1) if nz.numel() else (0, 0)
        starts.append(s)
        runs.append(table[p, s:e])
    S = max(1, max(r.numel() for r in runs))
    taps = torch.zeros(n, S, dtype=torch.float32)
    for p, r in enumerate(runs):
        taps[p, :r.numel()] = r
    return taps, torch.tensor(starts, dtype=torch.int32)


def delay_blocks(orig: int, new: int) -> int:
    o, _, width = reduced(orig, new)
    return -(-width // o)


def carry_samples(orig: int, new: int) -> int:
    o, _, width = reduced(orig, new)
    return delay_blocks(orig, new) * o + width


def streaming(x: torch.Tensor, orig: int, new: int) -> torch.Tensor:
    """What a StreamingResampler returns over chunks that concatenate to x [B, T] (T a multiple of o): the batch
    transform of [D * o zeros, x], first T / o * n samples."""
    o, n, _ = reduced(orig, new)
    D = delay_blocks(orig, new)
    z = torch.cat([torch.zeros(x.shape[0], D * o, dtype=x.dtype), x], dim=1)
    return resample(z, orig, new)[:, : x.shape[1] // o * n]


def run_sums64(x: torch.Tensor, taps: torch.Tensor, start: torch.Tensor, o: int, n: int, x_shift: int, out_len: int):
    """Per output of the kernel's definition (rows of x [R, L]): (float64 sum of the same fp32 operands over the phase's
    run, sum |x * h| in float64).  Both [R, out_len]."""
    R, L = x.shape
    S = taps.shape[1]
    q = torch.arange(out_len)
    j, p = q // n, q % n
    idx = (j * o + x_shift + start.long()[p])[:, None] + torch.arange(S)[None]          # [out_len, S]
    valid = (idx >= 0) & (idx < L)
    xv = x.double()[:, idx.clamp(0, max(L - 1, 0))] * valid                                # [R, out_len, S]
    h = taps.double()[p]                                                                  # [out_len, S]
    prod = xv * h
    return prod.sum(-1), prod.abs().sum(-1)


def seeded_input(rows: int, length: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return 0.3 * torch.randn(rows, length, generator=g)


def sha256(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()
