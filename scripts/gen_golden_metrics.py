"""Write tests/golden/codec_metrics.npz from the reference's own MultiResolutionSTFTLoss (a CPU box with the reference
sources; needs no GPU):

    python scripts/gen_golden_metrics.py --reference <RSTnet checkout>

Evaluation/codec/compute_ms_stft_loss.py is loaded unmodified, with a stub `librosa` module in sys.modules (the classes do
not use it) and its `torch.stft` call routed through a shim that passes return_complex=True and returns view_as_real (the
form the script was written for; current torch raises without return_complex).  The classes run in float64, with each
window buffer set to torch.hann_window(win) built in float64.  Per clip the file keeps (sc, mag) of every resolution and
their means, and asserts first that tests/metrics_oracle.py agrees to 1e-12.  Clips are not stored: they are
regenerated from their seeds (tests/metrics_oracle.py golden_pair), whose SHA-256 the file keeps.  Nothing of the
reference is copied.
"""
from __future__ import annotations

import argparse
import importlib.util
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import metrics_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "codec_metrics.npz")
# (length, seed, silent): 1025 = 2048 / 2 + 1, the shortest clip every resolution accepts; a length that is no multiple
# of any hop; one with long silent stretches (bins at the clamp floor); two seconds
CLIPS = ((1025, 11, False), (4321, 12, False), (24000, 13, True), (32000, 14, False))


class _TorchShim(types.ModuleType):
    """`torch` for the reference module: stft(..., return_complex=True) returned as view_as_real; everything else torch."""

    def __init__(self):
        super().__init__("torch")

    def __getattr__(self, name):
        return getattr(torch, name)

    @staticmethod
    def stft(*args, **kwargs):
        return torch.view_as_real(torch.stft(*args, return_complex=True, **kwargs))


def load_reference(root: str):
    path = os.path.join(root, "Evaluation", "codec", "compute_ms_stft_loss.py")
    for stub in ("librosa", "tqdm"):
        if stub not in sys.modules:
            try:
                __import__(stub)
            except ImportError:
                m = types.ModuleType(stub)
                if stub == "tqdm":
                    m.tqdm = lambda x, *a, **k: x
                sys.modules[stub] = m
    spec = importlib.util.spec_from_file_location("ref_compute_ms_stft_loss", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.torch = _TorchShim()
    return mod


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="root of the RSTnet sources (holds Evaluation/codec)")
    args = ap.parse_args()
    ref_mod = load_reference(args.reference)
    crit = ref_mod.MultiResolutionSTFTLoss().double()
    for layer in crit.loss_layers:
        layer.window = torch.hann_window(layer.win_size, dtype=torch.float64)
    resolutions = [(l.fft_size, l.hop_size, l.win_size) for l in crit.loss_layers]
    assert tuple(resolutions) == O.RESOLUTIONS, resolutions
    d = {"resolutions": np.array(resolutions, dtype=np.int64), "torch_version": np.array(torch.__version__)}
    d["lengths"] = np.array([c[0] for c in CLIPS], dtype=np.int64)
    d["seeds"] = np.array([c[1] for c in CLIPS], dtype=np.int64)
    d["silent"] = np.array([c[2] for c in CLIPS], dtype=np.bool_)
    per_res = np.zeros((len(CLIPS), len(resolutions), 2))
    total = np.zeros((len(CLIPS), 2))
    sha = []
    for i, (L, seed, silent) in enumerate(CLIPS):
        ref, deg = O.golden_pair(L, seed, silent)
        sha.append(O.sha256(ref, deg))
        fake, true = deg.double()[None], ref.double()[None]
        for j, layer in enumerate(crit.loss_layers):
            sc, mag = layer(fake, true)
            per_res[i, j] = (float(sc), float(mag))
            osc, omag = O.stft_loss(fake, true, *resolutions[j])
            assert abs(float(osc) - float(sc)) <= 1e-12 * abs(float(sc)) and abs(float(omag) - float(mag)) <= 1e-12 * abs(float(mag)), (L, j)
        sc, mag = crit(fake, true)
        total[i] = (float(sc), float(mag))
    d["sha256"] = np.array(sha)
    d["per_resolution"] = per_res
    d["total"] = total
    np.savez(OUT, **d)
    print(f"wrote {OUT}: {len(CLIPS)} clips")
    return 0


if __name__ == "__main__":
    sys.exit(main())
