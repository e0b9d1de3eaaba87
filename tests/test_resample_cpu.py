"""Resampling without a GPU: the CPU restatement of torchaudio.transforms.Resample against the torchaudio goldens, the
product's host table builder, the streaming arithmetic, the serving engine's rate check and the table cap."""
import math
import os

import numpy as np
import pytest
import torch

import resample_oracle as R
from rstnet_b200 import _lib, audio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# orig -> new: (o, n, K, w, min run, max run, delay blocks D) -- the table of the design notes
TABLE = {
    (16000, 24000): (2, 3, 16, 7, 12, 13, 4), (44100, 24000): (147, 80, 171, 12, 22, 23, 1),
    (48000, 24000): (2, 1, 28, 13, 25, 25, 7), (8000, 24000): (1, 3, 15, 7, 12, 13, 7),
    (22050, 24000): (147, 160, 161, 7, 12, 13, 1), (11025, 24000): (147, 320, 161, 7, 12, 13, 1),
    (24000, 16000): (3, 2, 23, 10, 18, 19, 4), (24000, 48000): (1, 2, 15, 7, 12, 13, 7),
    (24000, 8000): (3, 1, 41, 19, 37, 37, 7),
}


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "resample.npz"))


def _cases(g, key):
    for name in g[f"{key}__cases"]:
        base = f"{key}__{name}"
        rows, L = (int(v) for v in str(name)[1:].split("_L"))
        x = R.seeded_input(rows, L, int(g[f"{base}__seed"]))
        assert R.sha256(x) == str(g[f"{base}__x_sha256"]), f"input RNG drifted for {base}"
        yield x, torch.from_numpy(g[f"{base}__y"])


@pytest.mark.parametrize("pair", R.PAIRS)
def test_oracle_equals_torchaudio_goldens(golden, pair):
    key = "%d_%d" % pair
    kern, width = R.sinc_kernel(*pair)
    taps, start = R.trim(kern[:, 0])
    assert width == int(golden[f"{key}__width"]) and kern.shape[-1] == int(golden[f"{key}__K"])
    assert torch.equal(taps, torch.from_numpy(golden[f"{key}__taps"]))
    assert torch.equal(start, torch.from_numpy(golden[f"{key}__start"]))
    n_cases = 0
    for x, y in _cases(golden, key):
        assert torch.equal(R.resample(x, *pair), y)
        n_cases += 1
    assert n_cases >= 2                                           # lengths 1, o - 1, o (when distinct and > 0), ragged


@pytest.mark.parametrize("pair", R.PAIRS)
def test_host_table_equals_goldens(golden, pair):
    key = "%d_%d" % pair
    t = audio.resample_table(*pair)
    assert torch.equal(t.taps, torch.from_numpy(golden[f"{key}__taps"]))
    assert torch.equal(t.start, torch.from_numpy(golden[f"{key}__start"]))
    full, width = R.sinc_kernel(*pair)
    assert t.width == width and t.K == full.shape[-1]
    assert torch.equal(t.expand(), full[:, 0])                    # nothing outside the runs is lost
    runs = (t.taps != 0).sum(1)
    for p in range(t.n):                                          # each run is contiguous and its padded tail is zero
        assert bool((t.taps[p, :int(runs[p])] != 0).all()) and bool((t.taps[p, int(runs[p]):] == 0).all())
    o, n, K, w, rmin, rmax, D = TABLE[pair]
    assert (t.o, t.n, t.K, t.width, int(runs.min()), int(runs.max()), t.S) == (o, n, K, w, rmin, rmax, rmax)
    assert 4 * t.n * t.S <= audio.table_bytes_bound(*pair) <= _lib.RESAMPLE_MAX_TABLE_BYTES


@pytest.mark.parametrize("pair", R.PAIRS)
def test_streaming_arithmetic(pair):
    """Carry, delay and chunk arithmetic of StreamingResampler (no buffer is allocated before the first call)."""
    o, n, K, w, _, _, D = TABLE[pair]
    s = audio.StreamingResampler(*pair, batch=4, device="cpu")
    assert (s.o, s.n, s.width, s.delay_blocks) == (o, n, w, D)
    assert s.carry == D * o + w == R.carry_samples(*pair)
    assert s.latency_samples == D * n
    assert D * o >= w                                            # the carry covers the filter's look-ahead
    chunk = pair[0] * 2 // 25                                    # 80 ms
    assert chunk % o == 0 and s.output_length(chunk) == pair[1] * 2 // 25
    if o > 1:
        with pytest.raises(_lib.RstnetError, match="multiple"):
            s.output_length(chunk + 1)


def test_streaming_definition_matches_batch_oracle():
    """The streaming definition (zero prefix, then truncation) only needs the input seen so far: the first c chunks'
    output does not change when more input follows."""
    for orig, new in R.PAIRS:
        o = R.reduced(orig, new)[0]
        x = R.seeded_input(2, 6 * o * 7, 5)
        full = R.streaming(x, orig, new)
        part = R.streaming(x[:, : 3 * o * 7], orig, new)
        assert torch.equal(full[:, : part.shape[1]], part)


def test_engine_rate_check():
    from rstnet_b200.serve import check_client_rate
    for r in (8000, 11025, 16000, 22050, 32000, 44100, 48000, 24000):
        assert check_client_rate(r) == r
        if r != 24000:                                          # 80 ms is a whole number of blocks both ways
            assert (r * 2 // 25) % R.reduced(r, 24000)[0] == 0 and 1920 % R.reduced(24000, r)[0] == 0
            for pair in ((r, 24000), (24000, r)):               # and both tables fit the kernel's cap
                assert audio.table_bytes_bound(*pair) <= _lib.RESAMPLE_MAX_TABLE_BYTES
    for r in (24001, 12345, 0, -16000, 16000.5, "16000"):
        with pytest.raises(_lib.RstnetError, match="gcd"):
            check_client_rate(r)


def test_oversized_table_refused_before_allocation(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("the table was built")
    monkeypatch.setattr(audio, "sinc_table", boom)
    with pytest.raises(_lib.RstnetError, match="44100 Hz -> 24001 Hz"):
        audio.Resample(44100, 24001)
    with pytest.raises(_lib.RstnetError, match="44100 Hz -> 24001 Hz"):
        audio.StreamingResampler(44100, 24001, 4, "cpu")


def test_rate_validation_and_identity():
    for bad in ((16000.5, 24000), (16000, 0), (-1, 24000)):
        with pytest.raises(_lib.RstnetError):
            audio.Resample(*bad)
    x = torch.zeros(3)
    with pytest.raises(_lib.RstnetError, match="CUDA"):
        audio.Resample(24000, 24000)(x)                          # CPU input is refused even for the identity
    assert audio.Resample(24000, 24000).output_length(100) == 100
    assert audio.Resample(16000, 24000).output_length(7) == math.ceil(3 * 7 / 2)


def test_product_does_not_import_torchaudio():
    pkg = os.path.join(ROOT, "rstnet_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert "import torchaudio" not in src and "from torchaudio" not in src, f
