"""Write tests/golden/resample.npz from torchaudio.transforms.Resample (needs torchaudio; run on a CPU box):

    python scripts/gen_golden_resample.py

Asserts first that the CPU restatement in tests/resample_oracle.py reproduces torchaudio bit for bit (table and output)
for every case it stores.  Inputs are not stored: they are regenerated from the seeds, whose SHA-256 the file keeps.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import resample_oracle as R  # noqa: E402
from specs import mimi_spec as S  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "resample.npz")


def main() -> int:
    import torchaudio
    from torchaudio.transforms import Resample
    assert torchaudio.__version__.split("+")[0] == R.TORCHAUDIO_VERSION, torchaudio.__version__
    torch.manual_seed(0)
    d = {"torchaudio_version": np.array(torchaudio.__version__)}
    seed = 1000
    for orig, new in R.PAIRS:
        key = f"{orig}_{new}"
        tr = Resample(orig, new)
        kern, width = R.sinc_kernel(orig, new)
        assert torch.equal(kern.view(-1), tr.kernel.view(-1)) and kern.dtype == tr.kernel.dtype and width == tr.width, key
        table = kern[:, 0]
        taps, start = R.trim(table)
        o, n, w = R.reduced(orig, new)
        d[f"{key}__taps"], d[f"{key}__start"] = taps.numpy(), start.numpy()
        d[f"{key}__K"], d[f"{key}__width"] = np.array(table.shape[1]), np.array(width)
        ragged = int(0.3 * orig) + 7 if (int(0.3 * orig) + 7) % o else int(0.3 * orig) + 8
        lengths = sorted({1, o - 1, o, ragged} - {0})
        cases = [(1, L) for L in lengths]
        if (orig, new) == (16000, 24000):
            cases.append((3, 1001))                                   # a 3-row batch
        names = []
        for rows, L in cases:
            seed += 1
            x = R.seeded_input(rows, L, seed)
            y = tr(x)
            y_oracle = R.resample(x, orig, new)
            assert torch.equal(y, y_oracle) and y.shape[-1] == -(-n * L // o), (key, rows, L)
            name = f"{key}__r{rows}_L{L}"
            d[f"{name}__seed"], d[f"{name}__x_sha256"], d[f"{name}__y"] = np.array(seed), np.array(R.sha256(x)), y.numpy()
            names.append(f"r{rows}_L{L}")
        d[f"{key}__cases"] = np.array(names)
    # end-to-end tokenization: one 16 kHz and one 44.1 kHz clip and their 24 kHz torchaudio resampling
    for orig, L, s in ((16000, 16000, 901), (44100, 22050, 902)):
        x = S.synthetic_audio(1, L, seed=s)[0, 0]
        y = Resample(orig, 24000)(x)
        assert torch.equal(y, R.resample(x, orig, 24000))
        d[f"clip{orig}__seed"], d[f"clip{orig}__x_sha256"], d[f"clip{orig}__y24k"] = np.array(s), np.array(R.sha256(x)), y.numpy()
    np.savez_compressed(OUT, **d)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(d)} arrays")
    return 0


if __name__ == "__main__":
    sys.exit(main())
