"""Codec evaluation without a GPU: the float64 oracle against the reference's own MultiResolutionSTFTLoss
(tests/golden/codec_metrics.npz, scripts/gen_golden_metrics.py), SI-SNR identities, the C ABI symbols and the
`offline evaluate` command's arguments and file pairing."""
import math
import os

import numpy as np
import pytest
import torch

import metrics_oracle as O
from rstnet_b200 import _lib, offline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("rstnet_stft_loss_workspace", "rstnet_stft_loss_sums_f32", "rstnet_sisnr_moments_workspace",
               "rstnet_sisnr_moments_f32")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "codec_metrics.npz"))


def test_oracle_matches_reference_classes(golden):
    assert tuple(map(tuple, golden["resolutions"].tolist())) == O.RESOLUTIONS
    for i, (L, seed, silent) in enumerate(zip(golden["lengths"], golden["seeds"], golden["silent"])):
        ref, deg = O.golden_pair(int(L), int(seed), bool(silent))
        assert O.sha256(ref, deg) == str(golden["sha256"][i]), "golden clip RNG drifted"
        fake, true = deg.double()[None], ref.double()[None]
        for j, res in enumerate(O.RESOLUTIONS):
            sc, mag = O.stft_loss(fake, true, *res)
            np.testing.assert_allclose([float(sc), float(mag)], golden["per_resolution"][i, j], rtol=1e-12)
        sc, mag = O.ms_stft_loss(fake, true)
        np.testing.assert_allclose([float(sc), float(mag)], golden["total"][i], rtol=1e-12)
    assert int(golden["lengths"].min()) == 2048 // 2 + 1           # the shortest clip every resolution accepts
    assert bool(golden["silent"].any())


def test_silent_clip_reaches_the_clamp_floor(golden):
    i = int(np.flatnonzero(golden["silent"])[0])
    ref, _ = O.golden_pair(int(golden["lengths"][i]), int(golden["seeds"][i]), True)
    T = O.magnitude(O.spectrum(ref.double()[None], 512, 50, 240))
    assert float((T == math.sqrt(O.FLOOR)).double().mean()) > 0.1


def test_sums_restate_the_losses():
    ref, deg = O.golden_pair(5000, 3)
    s = O.stft_sums(ref[None], deg[None], 1024, 120, 600)[0]
    sc, mag = O.stft_loss(deg[None], ref[None], 1024, 120, 600)
    frames, bins = 1 + 5000 // 120, 1024 // 2 + 1
    assert math.isclose(math.sqrt(s[0]) / math.sqrt(s[1]), float(sc), rel_tol=1e-13)
    assert math.isclose(float(s[2]) / (frames * bins), float(mag), rel_tol=1e-13)


def test_si_snr_identities():
    g = torch.Generator().manual_seed(4)
    r = torch.randn(3, 4000, generator=g, dtype=torch.float64)
    d = r + 0.1 * torch.randn(3, 4000, generator=g, dtype=torch.float64)
    base = O.si_snr(d, r)
    for k in (0.01, 3.0, -2.0):
        torch.testing.assert_close(O.si_snr(k * d, r), base, rtol=1e-10, atol=0)      # the estimate's scale
    torch.testing.assert_close(O.si_snr(d, 5.0 * r), base, rtol=1e-10, atol=0)        # the reference's scale
    torch.testing.assert_close(O.si_snr(d + 0.7, r - 0.3), base, rtol=1e-10, atol=0)  # offsets are removed
    assert torch.isinf(O.si_snr(r, r)).all() and (O.si_snr(r, r) > 0).all()
    assert torch.isnan(O.si_snr(d, torch.full_like(r, 0.25))).all()
    # 10 log10(|s|^2 / |e|^2) for an estimate s + e with e orthogonal to s
    s = torch.sin(torch.arange(1000, dtype=torch.float64))
    s = s - s.mean()
    e = torch.cos(torch.arange(1000, dtype=torch.float64))
    e = e - e.mean()
    e = e - (e @ s) / (s @ s) * s
    e = e * 0.1 * s.norm() / e.norm()
    assert math.isclose(float(O.si_snr((s + e)[None], s[None])[0]), 20.0, rel_tol=1e-10)


def test_symbols_declared_exported_and_listed():
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert f" {name}(" in header and name in _lib.SYMBOLS, name
    from rstnet_b200 import build
    build.build()
    lib = _lib.lib()
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name), name
    assert lib.rstnet_version() == 206
    assert _lib.STFT_FRAMES_PER_BLOCK == 16 and _lib.SISNR_SAMPLES_PER_BLOCK == 8192
    assert "#define RSTNET_STFT_FRAMES_PER_BLOCK 16" in header and "#define RSTNET_SISNR_SAMPLES_PER_BLOCK 8192" in header


def test_workspace_sizes():
    lib = _lib.lib()
    assert lib.rstnet_stft_loss_workspace(3, 1000, 50) == 3 * math.ceil((1 + 1000 // 50) / 16) * 3 * 8
    assert lib.rstnet_sisnr_moments_workspace(2, 8193) == 2 * 2 * 5 * 8
    assert lib.rstnet_stft_loss_workspace(1, 100, 0) < 0 and lib.rstnet_sisnr_moments_workspace(-1, 10) < 0


def test_python_checks_before_any_launch():
    from rstnet_b200 import metrics as M
    for bad in ((1000, 120, 600), (32, 8, 32), (8192, 120, 600), (1024, 120, 0), (1024, 120, 1025), (1024, 0, 600)):
        with pytest.raises(_lib.RstnetError):
            M.STFTLoss(bad[0], bad[1], bad[2])
    with pytest.raises(_lib.RstnetError, match="CUDA"):
        M.STFTLoss()(torch.zeros(1, 2000), torch.zeros(1, 2000))
    with pytest.raises(_lib.RstnetError, match="CUDA"):
        M.si_snr(torch.zeros(1, 20), torch.zeros(1, 20))
    with pytest.raises(_lib.RstnetError):
        list(M.evaluate_pairs([], capacity_samples=0))


def test_si_snr_from_moments_edge_cases():
    from rstnet_b200 import metrics as M
    r = torch.tensor([0.5, -0.25, 0.125, 1.0], dtype=torch.float64)
    mom = lambda a, b: torch.stack([a.sum(), b.sum(), (a * a).sum(), (b * b).sum(), (a * b).sum()])
    n = torch.tensor([4])
    assert math.isinf(float(M.si_snr_from_moments(mom(r, r)[None], n)[0]))
    assert math.isnan(float(M.si_snr_from_moments(mom(torch.full_like(r, 0.3), r)[None], n)[0]))
    assert math.isnan(float(M.si_snr_from_moments(torch.zeros(1, 5, dtype=torch.float64), torch.tensor([0]))[0]))
    d = r + torch.tensor([0.01, -0.02, 0.0, 0.005], dtype=torch.float64)
    assert math.isclose(float(M.si_snr_from_moments(mom(r, d)[None], n)[0]), float(O.si_snr(d[None], r[None])[0]),
                        rel_tol=1e-9)


def test_clip_metrics_and_summary():
    from rstnet_b200 import metrics as M
    sums = torch.tensor([[4.0, 16.0, 10.0], [1.0, 4.0, 20.0], [9.0, 9.0, 30.0]], dtype=torch.float64)
    mom = torch.tensor([0.0, 0.0, 1.0, 1.0, 1.0], dtype=torch.float64)
    m = M.clip_metrics(sums, mom, 4800)
    sc = (0.5 + 0.5 + 1.0) / 3
    mag = (10.0 / ((1 + 4800 // 120) * 513) + 20.0 / ((1 + 4800 // 240) * 1025) + 30.0 / ((1 + 4800 // 50) * 257)) / 3
    assert math.isclose(m["sc"], sc) and math.isclose(m["mag"], mag) and math.isclose(m["ms_stft"], sc + mag)
    assert not m["skipped"] and math.isinf(m["sisnr"])
    short = M.clip_metrics(torch.full((3, 3), float("nan"), dtype=torch.float64), mom, 1024)
    assert short["skipped"] and math.isnan(short["ms_stft"])
    s = M.corpus_summary({"a": m, "b": short, "c": dict(m, sisnr=float("nan"), ms_stft=1.0)})
    assert s["clips"] == 3 and s["stft_skipped"] == 1 and s["sisnr_skipped"] == 1
    assert math.isclose(s["ms_stft"], (sc + mag + 1.0) / 2) and math.isinf(s["sisnr"])


def _write(path, n=400):
    offline.write_wav(path, torch.zeros(n), 16000)


def test_evaluate_arguments():
    a = offline.build_parser().parse_args(["evaluate", "--ref-dir", "R", "--deg-dir", "D"])
    assert (a.cmd, a.ref_dir, a.deg_dir, a.sample_rate, a.output_file) == ("evaluate", "R", "D", 16000, "metrics.json")
    assert a.capacity_seconds > 0
    a = offline.build_parser().parse_args(["evaluate", "--ref-dir", "R", "--deg-dir", "D", "--sample-rate", "24000",
                                           "--capacity-seconds", "30", "--output-file", "m.json"])
    assert (a.sample_rate, a.capacity_seconds, a.output_file) == (24000, 30.0, "m.json")
    for bad in (["--capacity-seconds", "0"], ["--capacity-seconds", "-1"]):
        with pytest.raises(SystemExit):
            offline.build_parser().parse_args(["evaluate", "--ref-dir", "R", "--deg-dir", "D"] + bad)
    with pytest.raises(SystemExit):
        offline.build_parser().parse_args(["evaluate", "--ref-dir", "R"])


def test_file_pairing(tmp_path):
    ref, deg = tmp_path / "ref", tmp_path / "deg"
    ref.mkdir()
    deg.mkdir()
    for n in ("b.wav", "a.wav", "c.wav"):
        _write(str(ref / n))
    for n in ("a.wav", "b.wav", "notes.txt"):
        (deg / n).write_bytes(b"") if n.endswith(".txt") else _write(str(deg / n))
    pairs = offline.pair_files(str(ref), str(deg))
    assert [p[0] for p in pairs] == ["a.wav", "b.wav"]
    assert pairs[0][1] == os.path.join(str(ref), "a.wav") and pairs[0][2] == os.path.join(str(deg), "a.wav")


def test_missing_reference_is_an_error_naming_the_files(tmp_path):
    ref, deg = tmp_path / "ref", tmp_path / "deg"
    ref.mkdir()
    deg.mkdir()
    _write(str(ref / "a.wav"))
    for n in ("a.wav", "x.wav", "y.wav"):
        _write(str(deg / n))
    with pytest.raises(FileNotFoundError, match=r"2 degraded.*x\.wav, y\.wav"):
        offline.pair_files(str(ref), str(deg))
    with pytest.raises(FileNotFoundError, match="x.wav"):
        offline.main(["evaluate", "--ref-dir", str(ref), "--deg-dir", str(deg), "--output-file", str(tmp_path / "m.json")])
    empty = tmp_path / "empty"
    empty.mkdir()
    with pytest.raises(FileNotFoundError, match="no wavs"):
        offline.pair_files(str(ref), str(empty))
