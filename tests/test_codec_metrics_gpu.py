"""GPU tests (-m gpu) of the codec evaluation kernels and their Python layer: the fused STFT-pair sums against the float64
oracle within an fp32 FFT error bound, SI-SNR moments, bit-identity across packings, NaN isolation, argument checks,
MultiResolutionSTFTLoss on a batch and `offline evaluate` end to end.

The bound.  The kernel computes, per frame, one radix-2 FFT of N points in fp32 with twiddles rounded once from fp64.
For such an FFT, ||Z^ - Z||_2 <= log2(N) * eta * ||Z||_2 with eta = mu + gamma_4 (sqrt(2) + mu) ~ 6.7 u (Higham,
"Accuracy and Stability of Numerical Algorithms", 2nd ed., Thm. 24.2; u = 2^-24, mu <= u the twiddle error).  We take
eps = (log2(N) + 2) * 8 u: the two extra terms cover the window product on input and the separation of the two spectra
(one addition and one halving).  ||Z||_2 = sqrt(N) ||z||_2 for the frame z = w r + i w d, so every bin's complex error, and
therefore its magnitude error (the clamp and sqrt(max(m^2, floor)) = max(m, sqrt floor) are 1-Lipschitz), is at most
delta_f = eps sqrt(N) ||z_f||_2.  Then, with E = 2 sqrt(bins * sum_f delta_f^2):
  |sqrt(S0^) - ||T - P||| <= E,   |sqrt(S1^) - ||T||| <= E / 2,
  |S2^ - S2| <= sum over bins of log((T + d) / max(T - d, floor)) + the same for P.
The kernel's fp64 sums add rounding far below these.  As a check that the bound is an FFT bound and not one fitted to
this kernel, CPU fp32 torch.stft on the same inputs must lie inside it too."""
import math
import os

import numpy as np
import pytest
import torch

import metrics_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
SQFLOOR = math.sqrt(O.FLOOR)


def _frame_norms(ref, deg, n_fft, hop, win):
    """||z_f||_2 of every frame of the windowed pair, float64 [frames] (torch.stft's framing)."""
    w = torch.zeros(n_fft, dtype=torch.float64)
    left = (n_fft - win) // 2
    w[left:left + win] = torch.hann_window(win, dtype=torch.float64)
    pad = lambda x: torch.nn.functional.pad(x.double()[None, None], (n_fft // 2, n_fft // 2), mode="reflect")[0, 0]
    fr = pad(ref).unfold(0, n_fft, hop) * w
    fd = pad(deg).unfold(0, n_fft, hop) * w
    return torch.sqrt((fr * fr).sum(1) + (fd * fd).sum(1))


def bound(ref, deg, n_fft, hop, win):
    """(exact fp64 sums [3], E, S2 bound) of one clip."""
    eps = (math.log2(n_fft) + 2) * 8 * U
    delta = eps * math.sqrt(n_fft) * _frame_norms(ref, deg, n_fft, hop, win)[:, None]        # [frames, 1]
    T = O.magnitude(O.spectrum(ref[None], n_fft, hop, win))[0]
    P = O.magnitude(O.spectrum(deg[None], n_fft, hop, win))[0]
    bins = n_fft // 2 + 1
    E = 2 * math.sqrt(bins * float((delta ** 2).sum()))
    dev = lambda M: torch.log((M + delta) / torch.clamp(M - delta, min=SQFLOOR)).sum()
    sums = torch.stack([((T - P) ** 2).sum(), (T ** 2).sum(), (P.log() - T.log()).abs().sum()])
    return sums, E, float(dev(T) + dev(P))


def assert_within(got, ref, deg, res, what=""):
    exact, E, S2b = bound(ref, deg, *res)
    got = [float(v) for v in got]
    slack = 1e-12
    assert abs(math.sqrt(got[0]) - math.sqrt(float(exact[0]))) <= E + slack, (what, got, exact, E)
    assert abs(math.sqrt(got[1]) - math.sqrt(float(exact[1]))) <= E / 2 + slack, (what, got, exact, E)
    assert abs(got[2] - float(exact[2])) <= S2b + slack * float(exact[2]), (what, got, exact, S2b)


def _pack(clips, gap=0, dev=DEV):
    """Pack [(ref, deg)] into buffers with `gap` unused samples before each clip -> (ref, deg, offsets, lengths)."""
    offs, parts_r, parts_d, pos = [], [], [], 0
    for r, d in clips:
        parts_r += [torch.full((gap,), 7.0), r]
        parts_d += [torch.full((gap,), -7.0), d]
        offs.append(pos + gap)
        pos += gap + r.numel()
    R = torch.cat(parts_r).to(dev)
    D = torch.cat(parts_d).to(dev)
    lens = [r.numel() for r, _ in clips]
    return R, D, torch.tensor(offs, device=dev), torch.tensor(lens, device=dev), lens


def _sums(clips, res, gap=0):
    from rstnet_b200 import metrics as M
    R, D, off, ln, lens = _pack(clips, gap)
    return M.stft_sums(R, D, off, ln, min(lens), max(lens), res).cpu()


def _moments(clips, gap=0):
    from rstnet_b200 import metrics as M
    R, D, off, ln, lens = _pack(clips, gap)
    return M.sisnr_moments(R, D, off, ln, max(lens)).cpu()


# (n_fft, hop, win, L, kind)
CASES = [
    (1024, 120, 600, 37123, "noise"), (2048, 240, 1200, 37123, "noise"), (512, 50, 240, 37123, "noise"),
    (2048, 240, 1200, 1025, "noise"),            # L = n_fft / 2 + 1
    (512, 50, 240, 257, "noise"),
    (1024, 120, 600, 16001, "noise"),            # L not a multiple of hop
    (256, 300, 200, 5000, "noise"),              # hop > win
    (1024, 120, 601, 9001, "noise"),             # odd n_fft - win
    (512, 128, 512, 7000, "noise"),              # win = n_fft
    (64, 16, 64, 1000, "noise"), (4096, 1024, 4096, 12000, "noise"),
    (1024, 120, 600, 20000, "silent"),
    (1024, 120, 600, 640000, "noise"),           # 40 s at 16 kHz
    (512, 50, 240, 640000, "gated"),
]


def _clip(L, kind, seed=0):
    if kind == "silent":
        return torch.zeros(L), torch.zeros(L)
    return O.golden_pair(L, 100 + seed + L % 997, silent=(kind == "gated"))


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"n{c[0]}_h{c[1]}_w{c[2]}_L{c[3]}_{c[4]}")
def test_kernel_sums_within_fp32_bound(case):
    n_fft, hop, win, L, kind = case
    r, d = _clip(L, kind)
    got = _sums([(r, d)], (n_fft, hop, win))[0]
    assert_within(got, r, d, (n_fft, hop, win), "gpu")
    if kind == "silent":                                               # every bin at the floor: exact
        bins, frames = n_fft // 2 + 1, 1 + L // hop
        assert float(got[0]) == 0.0 and float(got[2]) == 0.0
        assert math.isclose(float(got[1]), frames * bins * O.FLOOR, rel_tol=1e-12)
    if L <= 40000:                                                     # the bound is an fp32 FFT bound: CPU fp32 passes too
        win32 = torch.hann_window(win)
        T = torch.stft(r[None], n_fft, hop, win, win32, return_complex=True)[0].abs().double()
        P = torch.stft(d[None], n_fft, hop, win, win32, return_complex=True)[0].abs().double()
        T, P = T.clamp(min=SQFLOOR), P.clamp(min=SQFLOOR)
        assert_within([((T - P) ** 2).sum(), (T ** 2).sum(), (P.log() - T.log()).abs().sum()], r, d, (n_fft, hop, win),
                      "cpu fp32")


def test_golden_clips_match_reference_through_oracle(golden_dir):
    """GPU sc / mag per resolution of the golden clips against the reference classes' values, within the bound."""
    g = np.load(os.path.join(golden_dir, "codec_metrics.npz"))
    for i, (L, seed, silent) in enumerate(zip(g["lengths"], g["seeds"], g["silent"])):
        r, d = O.golden_pair(int(L), int(seed), bool(silent))
        for j, res in enumerate(O.RESOLUTIONS):
            got = _sums([(r, d)], res)[0]
            assert_within(got, r, d, res, f"golden {i} res {j}")
            exact, E, S2b = bound(r, d, *res)
            num, den = math.sqrt(float(got[0])), math.sqrt(float(got[1]))
            sc_ref, mag_ref = g["per_resolution"][i, j]
            en, ed = math.sqrt(float(exact[0])), math.sqrt(float(exact[1]))
            assert (en - E) / (ed + E / 2) - 1e-12 <= num / den <= (en + E) / (ed - E / 2) + 1e-12
            assert abs(en / ed - sc_ref) <= 1e-11 * sc_ref
            count = (1 + int(L) // res[1]) * (res[0] // 2 + 1)
            assert abs(float(got[2]) / count - mag_ref) <= S2b / count + 1e-11 * mag_ref


def _corpus():
    lens = [640000, 1025, 30011, 8192, 8193, 161, 99999]
    return [O.golden_pair(L, 900 + i, silent=(i == 2)) for i, L in enumerate(lens)]


def test_bit_identity_across_packings():
    clips = _corpus()
    long_ = [c for c in clips if c[0].numel() > 1024]
    for res in O.RESOLUTIONS:
        elig = [c for c in clips if c[0].numel() > res[0] // 2]
        base = _sums(elig, res)
        alone = torch.cat([_sums([c], res) for c in elig])
        rev = _sums(elig[::-1], res).flip(0)
        gapped = _sums(elig, res, gap=333)
        for other in (alone, rev, gapped):
            assert base.numpy().tobytes() == other.numpy().tobytes(), res
        sub = _sums(long_[1:3], res)                                   # another pack's min_len / max_len
        idx = [i for i, c in enumerate(elig) if any(c is x for x in long_[1:3])]
        assert base[idx].numpy().tobytes() == sub.numpy().tobytes()
    mb = _moments(clips)
    for other in (torch.cat([_moments([c]) for c in clips]), _moments(clips[::-1]).flip(0), _moments(clips, gap=5)):
        assert mb.numpy().tobytes() == other.numpy().tobytes()


def test_evaluate_pairs_independent_of_capacity_and_order():
    from rstnet_b200 import metrics as M
    clips = _corpus()
    items = [(f"c{i}", r, 16000, d, 16000) for i, (r, d) in enumerate(clips)]
    runs = [dict(M.evaluate_pairs(items, 16000, cap)) for cap in (1 << 24, 700000, 50000, 1)]
    runs.append(dict(M.evaluate_pairs(items[::-1], 16000, 123456)))
    for run in runs[1:]:
        assert set(run) == set(runs[0])
        for k, m in runs[0].items():
            a, b = np.array([m[x] for x in ("sisnr", "sc", "mag", "ms_stft")]), \
                np.array([run[k][x] for x in ("sisnr", "sc", "mag", "ms_stft")])
            assert a.tobytes() == b.tobytes(), k
    m = runs[0]
    assert m["c5"]["skipped"] and math.isnan(m["c5"]["ms_stft"]) and math.isfinite(m["c5"]["sisnr"])   # 161 samples
    assert not m["c1"]["skipped"]                                                                      # 1025 samples
    # per clip against the oracle
    for i, (r, d) in enumerate(clips):
        assert math.isclose(m[f"c{i}"]["sisnr"], float(O.si_snr(d[None], r[None])[0]), rel_tol=1e-9)


def test_nan_clip_leaves_others_untouched():
    clips = _corpus()[:4]
    bad_r = clips[2][0].clone()
    bad_r[12345] = float("nan")
    poisoned = clips[:2] + [(bad_r, clips[2][1])] + clips[3:]
    for res in O.RESOLUTIONS:
        a, b = _sums(clips, res), _sums(poisoned, res)
        keep = [0, 1, 3] if clips[1][0].numel() > res[0] // 2 else [0, 3]
        assert a[keep].numpy().tobytes() == b[keep].numpy().tobytes()
        assert torch.isnan(b[2]).all()
    a, b = _moments(clips), _moments(poisoned)
    assert a[[0, 1, 3]].numpy().tobytes() == b[[0, 1, 3]].numpy().tobytes() and torch.isnan(b[2]).any()


def test_argument_checks_are_error_returns():
    from rstnet_b200 import _lib, ops
    from rstnet_b200 import metrics as M
    r = torch.randn(4000, device=DEV)
    off = torch.zeros(1, dtype=torch.int64, device=DEV)
    ln = torch.full((1,), 4000, dtype=torch.int64, device=DEV)
    out = torch.zeros(1, 3, dtype=torch.float64, device=DEV)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=DEV)
    tw, w = M.stft_tables(1024, 600, DEV)
    good = dict(min_len=4000, max_len=4000, n_fft=1024, hop=120, win=600, n_res=1, res=0)
    for change, msg in ((dict(n_fft=1000), "power of two"), (dict(n_fft=32), "power of two"), (dict(n_fft=8192), "power of two"),
                        (dict(win=0), "win_length"), (dict(win=1025), "win_length"), (dict(hop=0), "hop"),
                        (dict(min_len=512), "n_fft / 2"), (dict(max_len=3999), "n_fft / 2"), (dict(res=1), "resolution")):
        a = dict(good, **change)
        with pytest.raises(_lib.RstnetError, match=msg):
            ops.stft_loss_sums(r, r, off, ln, 1, a["min_len"], a["max_len"], a["n_fft"], a["hop"], a["win"], tw, w, out,
                               a["n_res"], a["res"], ws)
    with pytest.raises(_lib.RstnetError, match="workspace"):
        ops.stft_loss_sums(r, r, off, ln, 1, 4000, 4000, 1024, 120, 600, tw, w, out, 1, 0, ws[:8])
    with pytest.raises(_lib.RstnetError, match="workspace"):
        ops.sisnr_moments(r, r, off, ln, 1, 4000, torch.zeros(1, 5, dtype=torch.float64, device=DEV), ws[:8])
    lib = _lib.lib()
    assert lib.rstnet_stft_loss_sums_f32(None, None, None, None, 1, 4000, 4000, 1024, 120, 600, None, None, None, 1, 0,
                                         None, 0, None) != 0
    assert b"null" in lib.rstnet_last_error()
    torch.cuda.synchronize()
    assert float(out.abs().sum()) == 0.0                                  # nothing was launched
    with pytest.raises(_lib.RstnetError, match="too short"):
        M.STFTLoss(2048, 240, 1200)(torch.zeros(2, 1024, device=DEV), torch.zeros(2, 1024, device=DEV))


def test_lengths_outside_the_promise_give_nan():
    from rstnet_b200 import metrics as M
    r, d = O.golden_pair(5000, 1)
    R, D, off, ln, _ = _pack([(r, d), (r, d)])
    s = M.stft_sums(R, D, off, ln, 5000, 4999 + 1, (1024, 120, 600)).cpu()
    assert torch.isfinite(s).all()
    ln2 = torch.tensor([5000, 6000], device=DEV)
    R2, D2 = torch.cat([R, torch.zeros(1000, device=DEV)]), torch.cat([D, torch.zeros(1000, device=DEV)])
    s2 = M.stft_sums(R2, D2, off, ln2, 5000, 5000, (1024, 120, 600)).cpu()
    assert s2[0].numpy().tobytes() == s[0].numpy().tobytes() and torch.isnan(s2[1]).all()


def test_multi_resolution_loss_on_a_batch():
    from rstnet_b200 import metrics as M
    B, L = 5, 24007
    pairs = [O.golden_pair(L, 300 + b, silent=(b == 3)) for b in range(B)]
    true = torch.stack([p[0] for p in pairs])
    fake = torch.stack([p[1] for p in pairs])
    crit = M.MultiResolutionSTFTLoss()
    sc, mag = crit(fake.to(DEV), true.to(DEV))
    assert sc.dtype == torch.float32 and sc.dim() == 0 and sc.is_cuda
    osc, omag = O.ms_stft_loss(fake.double(), true.double())
    sc_lo = sc_hi = mag_b = 0.0
    for res in O.RESOLUTIONS:
        ex, Es, S2s = zip(*(bound(t, f, *res) for t, f in zip(true, fake)))
        exact = torch.stack(ex).sum(0)
        E = math.sqrt(sum(e * e for e in Es))                          # the perturbation norms add in quadrature
        en, ed = math.sqrt(float(exact[0])), math.sqrt(float(exact[1]))
        sc_lo += (en - E) / (ed + E / 2) / 3
        sc_hi += (en + E) / (ed - E / 2) / 3
        mag_b += sum(S2s) / (B * (1 + L // res[1]) * (res[0] // 2 + 1)) / 3
    f32 = 2.0 ** -23                                                   # the fp32 result's rounding
    assert sc_lo * (1 - f32) <= float(sc) <= sc_hi * (1 + f32) and sc_lo <= float(osc) <= sc_hi
    assert abs(float(mag) - float(omag)) <= mag_b + f32 * float(omag)


def test_si_snr_gpu():
    from rstnet_b200 import metrics as M
    g = torch.Generator().manual_seed(8)
    r = torch.randn(4, 30000, generator=g) * 0.1 + 0.02
    d = r + 0.05 * torch.randn(4, 30000, generator=g)
    got = M.si_snr(d.to(DEV), r.to(DEV)).cpu()
    torch.testing.assert_close(got, O.si_snr(d, r), rtol=1e-9, atol=0)
    assert torch.isinf(M.si_snr(r.to(DEV), r.to(DEV))).all()
    assert torch.isnan(M.si_snr(d.to(DEV), torch.full_like(r, 0.3).to(DEV))).all()
    s2 = M.si_snr((4.0 * d).to(DEV), r.to(DEV)).cpu()                  # x4 is exact in fp32
    torch.testing.assert_close(s2, got, rtol=1e-9, atol=0)


def test_offline_evaluate_end_to_end(tmp_path, official_weights, capsys):
    import json
    from rstnet_b200 import offline
    from rstnet_b200.codec import MimiCodec
    from specs import mimi_spec as S
    src, dst = tmp_path / "ref", tmp_path / "rec"
    src.mkdir()
    for i, L in enumerate((28800, 12000, 48000)):
        offline.write_wav(str(src / f"u{i}.wav"), S.synthetic_audio(1, L, seed=60 + i)[0, 0], 24000)
    m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(official_weights, strict=True)
    m = m.to(DEV).eval()
    assert offline.reconstruct_directory(m, str(src), str(dst)) == 3
    out = tmp_path / "metrics.json"
    assert offline.main(["evaluate", "--ref-dir", str(src), "--deg-dir", str(dst), "--sample-rate", "24000",
                         "--capacity-seconds", "2.5", "--output-file", str(out)]) == 0
    printed = capsys.readouterr().out
    res = json.load(open(out))
    assert f"MS-STFT-Loss: {res['summary']['ms_stft']}" in printed and f"SI-SNR: {res['summary']['sisnr']}" in printed
    assert res["summary"]["clips"] == 3 and res["summary"]["stft_skipped"] == 0
    for name, mm in res["clips"].items():
        r, _ = offline.read_wav(str(src / name))
        d, _ = offline.read_wav(str(dst / name))
        L = min(r.numel(), d.numel())
        r, d = r[:L], d[:L]
        assert mm["samples"] == L
        osc, omag = O.ms_stft_loss(d.double()[None], r.double()[None])
        sc_b = mag_b = 0.0
        for res_ in O.RESOLUTIONS:
            exact, E, S2b = bound(r, d, *res_)
            en, ed = math.sqrt(float(exact[0])), math.sqrt(float(exact[1]))
            sc_b += max((en + E) / (ed - E / 2) - en / ed, en / ed - (en - E) / (ed + E / 2)) / 3
            mag_b += S2b / ((1 + L // res_[1]) * (res_[0] // 2 + 1)) / 3
        assert abs(mm["sc"] - float(osc)) <= sc_b + 1e-12 and abs(mm["mag"] - float(omag)) <= mag_b + 1e-12
        assert math.isclose(mm["sisnr"], float(O.si_snr(d[None], r[None])[0]), rel_tol=1e-9, abs_tol=1e-9)
    # every file against itself
    assert offline.main(["evaluate", "--ref-dir", str(src), "--deg-dir", str(src), "--sample-rate", "24000",
                         "--output-file", str(out)]) == 0
    res = json.load(open(out))
    for mm in res["clips"].values():
        assert mm["sc"] == 0.0 and mm["mag"] == 0.0 and mm["ms_stft"] == 0.0
        assert math.isinf(mm["sisnr"]) and mm["sisnr"] > 0
    # resampled: 24 kHz files scored at 16 kHz
    assert offline.main(["evaluate", "--ref-dir", str(src), "--deg-dir", str(dst), "--output-file", str(out)]) == 0
    res = json.load(open(out))
    assert res["sample_rate"] == 16000 and all(math.isfinite(mm["ms_stft"]) for mm in res["clips"].values())
