"""Float64 CPU restatement of the codec evaluation metrics (test infrastructure only; the product never imports it).

  * the multi-resolution STFT loss of Evaluation/codec/compute_ms_stft_loss.py: torch.stft(x, fft, hop, win,
    hann_window(win)) with the call's defaults (center=True, reflect padding, the window zero-padded centred to fft,
    onesided, not normalised), through `return_complex=True` in float64; magnitude sqrt(clamp(re^2 + im^2, min=1e-7));
    SpectralConvergence = ||T - P||_F / ||T||_F and LogSTFTMagnitude = mean |log P - log T|, T from the true (reference)
    signal and P from the fake (degraded) one; each averaged over the resolutions.
  * SI-SNR (Le Roux et al. 2019) on mean-removed signals, without an epsilon.

scripts/gen_golden_metrics.py pins the STFT part to the reference classes themselves (tests/golden/codec_metrics.npz).
"""
from __future__ import annotations

import hashlib

import torch

RESOLUTIONS = ((1024, 120, 600), (2048, 240, 1200), (512, 50, 240))   # (fft, hop, win)
FLOOR = 1e-7


def spectrum(x: torch.Tensor, n_fft: int, hop: int, win: int) -> torch.Tensor:
    """complex128 [B, frames, bins] of x [B, L]."""
    x = x.to(torch.float64)
    s = torch.stft(x, n_fft, hop, win, torch.hann_window(win, dtype=torch.float64), return_complex=True)
    return s.transpose(2, 1)


def magnitude(spec: torch.Tensor) -> torch.Tensor:
    return torch.sqrt(torch.clamp(spec.real ** 2 + spec.imag ** 2, min=FLOOR))


def stft_sums(ref: torch.Tensor, deg: torch.Tensor, n_fft: int, hop: int, win: int) -> torch.Tensor:
    """float64 [B, 3] per row: sum (T - P)^2, sum T^2, sum |log P - log T| (what rstnet_stft_loss_sums_f32 computes)."""
    T = magnitude(spectrum(ref, n_fft, hop, win))
    P = magnitude(spectrum(deg, n_fft, hop, win))
    return torch.stack([((T - P) ** 2).sum((1, 2)), (T ** 2).sum((1, 2)), (P.log() - T.log()).abs().sum((1, 2))], dim=1)


def stft_loss(fake: torch.Tensor, true: torch.Tensor, n_fft: int, hop: int, win: int):
    """(sc, mag) of STFTLoss over the batch [B, L]: the norms and the mean run over the whole [B, frames, bins] tensor."""
    T = magnitude(spectrum(true, n_fft, hop, win))
    P = magnitude(spectrum(fake, n_fft, hop, win))
    return torch.linalg.norm((T - P).flatten()) / torch.linalg.norm(T.flatten()), (P.log() - T.log()).abs().mean()


def ms_stft_loss(fake: torch.Tensor, true: torch.Tensor, resolutions=RESOLUTIONS):
    scs, mags = zip(*(stft_loss(fake, true, *r) for r in resolutions))
    return sum(scs) / len(scs), sum(mags) / len(mags)


def si_snr(est: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    """float64 [B]: 10 log10(alpha^2 <r~, r~> / ||d~ - alpha r~||^2), alpha = <d~, r~> / <r~, r~>."""
    r = ref.to(torch.float64)
    d = est.to(torch.float64)
    r = r - r.mean(-1, keepdim=True)
    d = d - d.mean(-1, keepdim=True)
    alpha = (d * r).sum(-1) / (r * r).sum(-1)
    e = d - alpha[..., None] * r
    return 10.0 * torch.log10(alpha ** 2 * (r * r).sum(-1) / (e * e).sum(-1))


def golden_pair(L: int, seed: int, silent: bool = False):
    """A seeded (reference, degraded) fp32 pair of length L: a few sinusoids and noise; the degraded one is the reference
    scaled, with added noise and a short echo.  `silent`: long exact-zero stretches in both (the clamp floor)."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L, dtype=torch.float64) / 16000.0
    freqs = torch.empty(4, dtype=torch.float64).uniform_(80.0, 6000.0, generator=g)
    amps = torch.empty(4, dtype=torch.float64).uniform_(0.02, 0.1, generator=g)
    ref = (amps[:, None] * torch.sin(2 * torch.pi * freqs[:, None] * t[None])).sum(0)
    ref = ref + 0.01 * torch.randn(L, generator=g, dtype=torch.float64)
    deg = 0.8 * ref + 0.02 * torch.randn(L, generator=g, dtype=torch.float64)
    deg[7:] += 0.1 * ref[:-7]
    if silent:
        gate = torch.zeros(L, dtype=torch.float64)
        for a in range(0, L, 8000):
            gate[a:a + 2500] = 1.0
        ref, deg = ref * gate, deg * gate
    return ref.to(torch.float32), deg.to(torch.float32)


def sha256(*ts) -> str:
    h = hashlib.sha256()
    for t in ts:
        h.update(t.contiguous().numpy().tobytes())
    return h.hexdigest()
