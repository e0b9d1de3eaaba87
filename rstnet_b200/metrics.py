"""Codec evaluation on the GPU: the multi-resolution STFT loss of the reference's Evaluation/codec/compute_ms_stft_loss.py
and SI-SNR, per clip, over whole corpora.

  * `STFTLoss(fft_size, hop_size, win_size)` / `MultiResolutionSTFTLoss(fft_sizes, win_sizes, hop_sizes)`: the reference
    classes (compute_ms_stft_loss.py:50-99) with their constructor arguments and defaults.  `forward(fake [B, L],
    true [B, L]) -> (sc_loss, mag_loss)` on CUDA fp32 tensors, with the reference's batch semantics: the Frobenius norm
    and the L1 mean run over the whole [B, frames, bins] tensor.  Each resolution is one fused kernel
    (`rstnet_stft_loss_sums_f32`): one complex FFT per frame gives both spectra, and the magnitudes are never stored, so
    `SpectralConvergence` / `LogSTFTMagnitude` (which take magnitudes) have no counterpart here.
  * `si_snr(est, ref)`: per-row SI-SNR in dB.  The reference imports `estimate_si_sdr` from a `sisnr` module that it
    does not ship, so the definition is this project's: the scale-invariant SNR of Le Roux et al. (2019, "SDR -
    half-baked or well done?") on mean-removed signals, without an epsilon.  With r~, d~ the mean-removed reference and
    estimate, alpha = <d~, r~> / <r~, r~> and SI-SNR = 10 log10(alpha^2 <r~, r~> / ||d~ - alpha r~||^2).  Identical
    signals give +inf; an all-constant reference gives NaN.
  * `evaluate_pairs(items, sample_rate, capacity_samples)`: every (key, ref_wav, ref_sr, deg_wav, deg_sr) item resampled
    to `sample_rate` (`audio.Resample`, torchaudio's defaults), both trimmed to the shorter length as the reference scripts
    do, and packed with other clips into launches of up to `capacity_samples` samples; yields (key, metrics) as packs
    finish.  A clip's numbers do not depend on its pack.

PESQ, STOI, ViSQOL, MCD, mel-SSIM and DNSMOS (the other scripts of Evaluation/codec) are not provided: each needs an
external package or model, so none could be pinned against an implementation here.

There is no CPU path: inputs must be CUDA fp32 tensors.
"""
from __future__ import annotations

import math
from typing import Dict, Iterable, Iterator, List, Optional, Sequence, Tuple

import torch

from . import _lib, ops
from ._lib import RstnetError
from .audio import Resample

# (fft_size, hop_size, win_size) of MultiResolutionSTFTLoss's defaults (compute_ms_stft_loss.py:79-81, 114-117)
RESOLUTIONS: Tuple[Tuple[int, int, int], ...] = ((1024, 120, 600), (2048, 240, 1200), (512, 50, 240))
DEFAULT_CAPACITY_SAMPLES = 1 << 24     # 17.5 min of 16 kHz audio per pack: 128 MB of ref + deg
# a centred reference energy below this fraction of sum r^2 is under the resolution of the fp64 moments (see si_snr_from_moments)
SISNR_CONSTANT_REF = 2.0 ** -40

_tables: Dict[tuple, Tuple[torch.Tensor, torch.Tensor]] = {}


def stft_tables(n_fft: int, win: int, device) -> Tuple[torch.Tensor, torch.Tensor]:
    """(twiddle fp32 [n_fft / 2, 2] = (cos, -sin)(2 pi k / n_fft), torch.hann_window(win) fp32), both computed in fp64 and
    rounded once, on `device`."""
    device = torch.device(device)
    key = (n_fft, win, device)
    if key not in _tables:
        k = torch.arange(n_fft // 2, dtype=torch.float64) * (2.0 * math.pi / n_fft)
        tw = torch.stack([torch.cos(k), -torch.sin(k)], dim=1).to(torch.float32)
        w = torch.hann_window(win, periodic=True, dtype=torch.float64).to(torch.float32)
        _tables[key] = (tw.contiguous().to(device), w.to(device))
    return _tables[key]


def _check_resolution(n_fft: int, hop: int, win: int) -> None:
    if not (64 <= n_fft <= 4096 and n_fft & (n_fft - 1) == 0):
        raise RstnetError(f"fft_size must be a power of two in [64, 4096], got {n_fft}")
    if not 1 <= win <= n_fft:
        raise RstnetError(f"win_size {win} outside [1, fft_size = {n_fft}]")
    if hop < 1:
        raise RstnetError(f"hop_size {hop} < 1")


def _check_input(x, what: str) -> None:
    if not isinstance(x, torch.Tensor):
        raise RstnetError(f"{what}: expected a torch.Tensor, got {type(x).__name__}")
    if not x.is_cuda:
        raise RstnetError(f"{what}: input must be a CUDA tensor (there is no CPU path)")
    if x.dtype != torch.float32:
        raise RstnetError(f"{what}: input must be float32, got {x.dtype}")


def stft_sums(ref: torch.Tensor, deg: torch.Tensor, offsets: torch.Tensor, lengths: torch.Tensor, min_len: int,
              max_len: int, resolution: Tuple[int, int, int], out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp64 [clips, 3]: (sum (T - P)^2, sum T^2, sum |log P - log T|) of one (fft, hop, win) resolution for the clips
    ref/deg[offsets[c] : offsets[c] + lengths[c]] of packed CUDA fp32 buffers (offsets / lengths: CUDA int64;
    min_len / max_len: bounds of the lengths, min_len > fft / 2)."""
    n_fft, hop, win = resolution
    _check_resolution(n_fft, hop, win)
    clips = int(lengths.numel())
    if out is None:
        out = torch.empty(clips, 3, dtype=torch.float64, device=ref.device)
    if clips == 0:
        return out
    tw, w = stft_tables(n_fft, win, ref.device)
    ws = torch.empty(max(1, ops.stft_loss_workspace(clips, max_len, hop)), dtype=torch.uint8, device=ref.device)
    ops.stft_loss_sums(ref, deg, offsets, lengths, clips, min_len, max_len, n_fft, hop, win, tw, w, out, 1, 0, ws)
    return out


def sisnr_moments(ref: torch.Tensor, deg: torch.Tensor, offsets: torch.Tensor, lengths: torch.Tensor,
                  max_len: int) -> torch.Tensor:
    """fp64 [clips, 5]: (sum r, sum d, sum r^2, sum d^2, sum r d) of the packed clips (as `stft_sums`)."""
    clips = int(lengths.numel())
    out = torch.empty(clips, 5, dtype=torch.float64, device=ref.device)
    if clips == 0:
        return out
    ws = torch.empty(max(1, ops.sisnr_moments_workspace(clips, max_len)), dtype=torch.uint8, device=ref.device)
    ops.sisnr_moments(ref, deg, offsets, lengths, clips, max_len, out, ws)
    return out


def si_snr_from_moments(m: torch.Tensor, n: torch.Tensor) -> torch.Tensor:
    """SI-SNR in dB of each row of m = (sum r, sum d, sum r^2, sum d^2, sum r d) over n samples, in fp64.

    With Srr = sum r^2 - (sum r)^2 / n (and Sdd, Srd alike), alpha = Srd / Srr and ||d~ - alpha r~||^2 = Sdd - alpha Srd.
    The moments are fp64 sums of exact products, each within about 60 * 2^-53 of its sum of magnitudes (at most ~50
    additions on any path of the fixed summation tree).  The denominator is a difference of such sums, so its error is
    about 2^-47 * (sum d^2 + sum r d); the SI-SNR stays within 0.05 dB of the exact value up to about 120 dB for signals
    whose mean is small beside their spread, and beyond that it is not resolved (it may read +inf).  A reference whose
    centred energy Srr is below 2^-40 sum r^2 is constant to within that resolution and gives NaN, as an exactly
    constant one does."""
    m = m.to(torch.float64)
    n = n.to(torch.float64)
    sr, sd, srr, sdd, srd = m.unbind(-1)
    Srr = srr - sr * sr / n
    Sdd = sdd - sd * sd / n
    Srd = srd - sr * sd / n
    const_ref = ~(Srr > SISNR_CONSTANT_REF * srr)
    alpha = Srd / Srr
    num = alpha * Srd
    den = (Sdd - alpha * Srd).clamp(min=0.0)     # identical signals: alpha == 1 and den == 0 exactly
    out = 10.0 * torch.log10(num / den)
    nan = torch.full_like(out, float("nan"))
    return torch.where(const_ref | (n <= 0), nan, out)


def si_snr(est: torch.Tensor, ref: torch.Tensor) -> torch.Tensor:
    """SI-SNR in dB of each row of est [B, L] against ref [B, L] (CUDA fp32): fp64 [B] on the same device."""
    _check_input(est, "si_snr")
    _check_input(ref, "si_snr")
    if est.shape != ref.shape or est.dim() != 2:
        raise RstnetError(f"si_snr: expected two [B, L] tensors of one shape, got {tuple(est.shape)} and {tuple(ref.shape)}")
    B, L = ref.shape
    r, d = ref.contiguous(), est.contiguous()
    offsets = torch.arange(B, dtype=torch.int64, device=r.device) * L
    lengths = torch.full((B,), L, dtype=torch.int64, device=r.device)
    m = sisnr_moments(r, d, offsets, lengths, L)
    return si_snr_from_moments(m, lengths)


class STFTLoss(torch.nn.Module):
    """compute_ms_stft_loss.py:50-73 on the GPU: forward(predicts [B, L], targets [B, L]) -> (sc_loss, mag_loss), 0-dim
    fp32 CUDA tensors (the sums are fp64)."""

    def __init__(self, fft_size: int = 1024, hop_size: int = 120, win_size: int = 600):
        super().__init__()
        _check_resolution(fft_size, hop_size, win_size)
        self.fft_size, self.hop_size, self.win_size = int(fft_size), int(hop_size), int(win_size)

    def sums(self, predicts: torch.Tensor, targets: torch.Tensor) -> Tuple[torch.Tensor, int]:
        """(fp64 [B, 3] per-row sums, elements per row = frames * bins)."""
        _check_input(predicts, "STFTLoss")
        _check_input(targets, "STFTLoss")
        if predicts.shape != targets.shape or predicts.dim() != 2:
            raise RstnetError(f"STFTLoss: expected two [B, L] tensors of one shape, got {tuple(predicts.shape)} and "
                              f"{tuple(targets.shape)}")
        B, L = targets.shape
        if L <= self.fft_size // 2:
            raise RstnetError(f"STFTLoss: signals of {L} samples are too short for fft_size {self.fft_size} "
                              f"(torch.stft's reflect padding needs more than {self.fft_size // 2})")
        t, p = targets.contiguous(), predicts.contiguous()
        offsets = torch.arange(B, dtype=torch.int64, device=t.device) * L
        lengths = torch.full((B,), L, dtype=torch.int64, device=t.device)
        s = stft_sums(t, p, offsets, lengths, L, L, (self.fft_size, self.hop_size, self.win_size))
        return s, (1 + L // self.hop_size) * (self.fft_size // 2 + 1)

    def forward(self, predicts: torch.Tensor, targets: torch.Tensor):
        s, per_row = self.sums(predicts, targets)
        tot = s.sum(dim=0)
        sc = tot[0].sqrt() / tot[1].sqrt()
        mag = tot[2] / (per_row * s.shape[0])
        return sc.to(torch.float32), mag.to(torch.float32)


class MultiResolutionSTFTLoss(torch.nn.Module):
    """compute_ms_stft_loss.py:76-99 on the GPU: the mean over resolutions of each STFTLoss's (sc_loss, mag_loss)."""

    def __init__(self, fft_sizes: Sequence[int] = (1024, 2048, 512), win_sizes: Sequence[int] = (600, 1200, 240),
                 hop_sizes: Sequence[int] = (120, 240, 50), **kwargs):
        super().__init__()
        self.loss_layers = torch.nn.ModuleList(
            STFTLoss(f, h, w) for f, w, h in zip(fft_sizes, win_sizes, hop_sizes))

    def forward(self, fake_signals: torch.Tensor, true_signals: torch.Tensor):
        sc, mag = zip(*(layer(fake_signals, true_signals) for layer in self.loss_layers))
        return sum(sc) / len(sc), sum(mag) / len(mag)


def _row(wav) -> torch.Tensor:
    wav = torch.as_tensor(wav)
    if wav.dim() == 2 and wav.shape[0] == 1:
        wav = wav[0]
    if wav.dim() != 1:
        raise RstnetError(f"expected mono audio [L] or [1, L], got {tuple(wav.shape)}")
    return wav.to(torch.float32)


def clip_metrics(sums: torch.Tensor, moments: torch.Tensor, L: int,
                 resolutions: Sequence[Tuple[int, int, int]] = RESOLUTIONS) -> dict:
    """One clip's metrics from its fp64 sums [n_res, 3] (NaN rows where it is too short) and moments [5]."""
    sc_r, mag_r = [], []
    for (n_fft, hop, _), (s0, s1, s2) in zip(resolutions, sums.tolist()):
        sc_r.append(math.sqrt(s0) / math.sqrt(s1) if s0 == s0 and s1 == s1 else float("nan"))
        mag_r.append(s2 / ((1 + L // hop) * (n_fft // 2 + 1)))
    skipped = L <= max(r[0] for r in resolutions) // 2
    nan = float("nan")
    sc = nan if skipped else sum(sc_r) / len(sc_r)
    mag = nan if skipped else sum(mag_r) / len(mag_r)
    sisnr = float(si_snr_from_moments(moments[None], torch.tensor([L]))[0])
    return {"sisnr": sisnr, "sc": sc, "mag": mag, "ms_stft": sc + mag, "skipped": skipped, "samples": L}


def _evaluate_pack(pack: List[Tuple[object, torch.Tensor, torch.Tensor]], resolutions) -> Iterator[Tuple[object, dict]]:
    dev = pack[0][1].device
    lens = [int(r.numel()) for _, r, _ in pack]
    ref = torch.cat([r for _, r, _ in pack])
    deg = torch.cat([d for _, _, d in pack])
    starts = [0]
    for L in lens[:-1]:
        starts.append(starts[-1] + L)
    offsets = torch.tensor(starts, dtype=torch.int64)
    lengths = torch.tensor(lens, dtype=torch.int64)
    sums = torch.full((len(pack), len(resolutions), 3), float("nan"), dtype=torch.float64)
    for i, res in enumerate(resolutions):
        idx = [c for c, L in enumerate(lens) if L > res[0] // 2]
        if not idx:
            continue
        sel = torch.tensor(idx, dtype=torch.int64)
        ls = [lens[c] for c in idx]
        s = stft_sums(ref, deg, offsets[sel].to(dev), lengths[sel].to(dev), min(ls), max(ls), res)
        sums[sel, i] = s.cpu()
    moments = sisnr_moments(ref, deg, offsets.to(dev), lengths.to(dev), max(lens)).cpu()
    for c, (key, _, _) in enumerate(pack):
        yield key, clip_metrics(sums[c], moments[c], lens[c], resolutions)


@torch.no_grad()
def evaluate_pairs(items: Iterable[Tuple], sample_rate: int = 16000, capacity_samples: int = DEFAULT_CAPACITY_SAMPLES,
                   device="cuda", resolutions: Sequence[Tuple[int, int, int]] = RESOLUTIONS) -> Iterator[Tuple[object, dict]]:
    """Yield (key, {"sisnr", "sc", "mag", "ms_stft", "skipped", "samples"}) for every (key, ref_wav, ref_sr, deg_wav, deg_sr)
    item, pack by pack.  Each signal is resampled to `sample_rate` and both are trimmed to the shorter length; clips are
    packed into launches of up to `capacity_samples` samples (a longer clip runs alone).  A clip too short for a
    resolution (L <= fft_size / 2) gets NaN STFT metrics and skipped = True, and still its SI-SNR; an empty clip is
    skipped entirely (every metric NaN).  `sc` and `mag` are the means over resolutions of the reference's per-clip
    SpectralConvergence and LogSTFTMagnitude, `ms_stft` = sc + mag (compute_ms_stft_loss.py:134-135)."""
    for r in resolutions:
        _check_resolution(*r)
    if capacity_samples < 1:
        raise RstnetError(f"capacity_samples must be >= 1, got {capacity_samples}")
    device = torch.device(device)
    resamplers: Dict[int, Resample] = {}

    def prep(wav, sr) -> torch.Tensor:
        w = _row(wav).to(device)
        sr = int(sr)
        if sr != sample_rate and w.numel():
            if sr not in resamplers:
                resamplers[sr] = Resample(sr, sample_rate)
            w = resamplers[sr](w)
        return w

    pack: List[Tuple[object, torch.Tensor, torch.Tensor]] = []
    filled = 0
    for key, ref_wav, ref_sr, deg_wav, deg_sr in items:
        r, d = prep(ref_wav, ref_sr), prep(deg_wav, deg_sr)
        L = min(r.numel(), d.numel())
        if L == 0:
            nan = float("nan")
            yield key, {"sisnr": nan, "sc": nan, "mag": nan, "ms_stft": nan, "skipped": True, "samples": 0}
            continue
        if pack and filled + L > capacity_samples:
            yield from _evaluate_pack(pack, resolutions)
            pack, filled = [], 0
        pack.append((key, r[:L], d[:L]))
        filled += L
    if pack:
        yield from _evaluate_pack(pack, resolutions)


def corpus_summary(metrics: Dict[object, dict]) -> dict:
    """Corpus means: the STFT metrics over clips not skipped, SI-SNR over clips whose SI-SNR is not NaN; with the counts of
    the clips left out of each."""
    stft = [m for m in metrics.values() if not m["skipped"]]
    sis = [m["sisnr"] for m in metrics.values() if m["sisnr"] == m["sisnr"]]
    mean = (lambda xs: sum(xs) / len(xs) if xs else float("nan"))
    return {"clips": len(metrics),
            "ms_stft": mean([m["ms_stft"] for m in stft]), "sc": mean([m["sc"] for m in stft]),
            "mag": mean([m["mag"] for m in stft]), "stft_skipped": len(metrics) - len(stft),
            "sisnr": mean(sis), "sisnr_skipped": len(metrics) - len(sis)}
