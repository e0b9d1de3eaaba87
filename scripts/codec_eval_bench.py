"""Throughput of codec evaluation (rstnet_b200.metrics.evaluate_pairs) on a seeded synthetic corpus (clip lengths uniform in
1 s .. 40 s, built as scripts/codec_corpus_bench.py builds its corpus, at 16 kHz; the degraded clip is the reference
scaled, with noise and an echo).  Prints one JSON line:

  * evaluate_pairs from device-resident audio: audio-seconds/s (host wall clock from a device synchronise to the last
    result on the host);
  * the same from 16-bit wav files on disk (a temporary directory; read_wav, upload and the pairing included) for the
    first --disk-clips clips;
  * kernel time of one pack per resolution and of the SI-SNR moments, from CUDA events over --reps launches;
  * the reference's way on the same corpus: per clip, fp32 torch.stft on the GPU at the three resolutions
    (compute_ms_stft_loss.py's STFTLoss arithmetic, return_complex=True), in the same run;
  * the largest per-clip difference in ms_stft between the two paths;
  * the card's name and power limit, read in the same call.

Shape arithmetic (not a measurement): per audio-second at 16 kHz the three resolutions take 134 + 67 + 321 frames of
1024-, 2048- and 512-point complex FFTs, 5 N log2 N flops each: about 22 MFLOP; the kernel reads each sample pair once
per resolution from HBM (8 B), 24 B over the three.

usage: python scripts/codec_eval_bench.py [--clips 1024] [--disk-clips 128] [--capacity-seconds 600] [--reps 20]
                                          [--seed 0] [--out FILE]
"""
import argparse
import json
import math
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rstnet_b200 import metrics as M            # noqa: E402
from rstnet_b200 import offline                 # noqa: E402
from specs import mimi_spec as S                # noqa: E402

SR = 16000


def corpus(n, seed):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1 * SR, 40 * SR + 1, size=n)
    out = []
    for i, L in enumerate(lengths):
        ref = S.synthetic_audio(1, int(L), seed=seed * 100003 + i)[0, 0]
        g = torch.Generator().manual_seed(seed * 100003 + i + 7)
        deg = 0.8 * ref + 0.01 * torch.randn(int(L), generator=g)
        deg[5:] += 0.1 * ref[:-5]
        out.append((f"utt{i:04d}", ref, deg))
    return out


def card():
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        q = f"nvidia-smi unavailable ({e})"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def reference_way(clips, dev):
    """Per clip, fp32 torch.stft on the GPU: STFTLoss of every resolution, then sc + mag (compute_ms_stft_loss.py)."""
    wins = {(f, w): torch.hann_window(w, device=dev) for f, _, w in M.RESOLUTIONS}
    out = {}
    for key, ref, deg in clips:
        r, d = ref.view(1, -1), deg.view(1, -1)
        sc = mag = 0.0
        for f, h, w in M.RESOLUTIONS:
            T = torch.stft(r, f, h, w, wins[(f, w)], return_complex=True)
            P = torch.stft(d, f, h, w, wins[(f, w)], return_complex=True)
            T = torch.sqrt(torch.clamp(T.real ** 2 + T.imag ** 2, min=1e-7))
            P = torch.sqrt(torch.clamp(P.real ** 2 + P.imag ** 2, min=1e-7))
            sc = sc + torch.norm(T - P, p="fro") / torch.norm(T, p="fro")
            mag = mag + torch.nn.functional.l1_loss(P.log(), T.log())
        out[key] = (sc + mag) / len(M.RESOLUTIONS)
    return {k: float(v) for k, v in out.items()}


def kernel_times(dev_clips, capacity, reps):
    """CUDA-event time of one pack (the first `capacity` samples' worth of clips) per resolution and for the moments."""
    pack, filled = [], 0
    for _, r, d in dev_clips:
        if pack and filled + r.numel() > capacity:
            break
        pack.append((r, d))
        filled += r.numel()
    ref = torch.cat([r for r, _ in pack])
    deg = torch.cat([d for _, d in pack])
    lens = [r.numel() for r, _ in pack]
    offsets = torch.tensor([0] + list(np.cumsum(lens)[:-1]), dtype=torch.int64, device=ref.device)
    lengths = torch.tensor(lens, dtype=torch.int64, device=ref.device)
    res = {"clips": len(pack), "audio_seconds": round(filled / SR, 1)}

    def ev(fn):
        fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / reps * 1e3     # us
    for f, h, w in M.RESOLUTIONS:
        out = torch.empty(len(lens), 3, dtype=torch.float64, device=ref.device)
        us = ev(lambda: M.stft_sums(ref, deg, offsets, lengths, min(lens), max(lens), (f, h, w), out))
        frames = sum(1 + L // h for L in lens)
        res[f"stft_{f}_{h}_{w}_us"] = round(us, 1)
        res[f"stft_{f}_{h}_{w}_gflops"] = round(frames * 5 * f * math.log2(f) / us / 1e3, 1)
        res[f"stft_{f}_{h}_{w}_GBps_min_traffic"] = round(8 * filled / us / 1e3, 1)
    res["moments_us"] = round(ev(lambda: M.sisnr_moments(ref, deg, offsets, lengths, max(lens))), 1)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1024)
    ap.add_argument("--disk-clips", type=int, default=128)
    ap.add_argument("--capacity-seconds", type=float, default=600.0)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = "cuda"
    cap = int(args.capacity_seconds * SR)
    clips = corpus(args.clips, args.seed)
    audio_s = sum(r.numel() for _, r, _ in clips) / SR
    res = {"card": card(), "clips": args.clips, "sample_rate": SR, "audio_seconds": round(audio_s, 1),
           "capacity_seconds": args.capacity_seconds}
    dev_clips = [(k, r.to(dev), d.to(dev)) for k, r, d in clips]
    items = [(k, r, SR, d, SR) for k, r, d in dev_clips]
    dict(M.evaluate_pairs(items[:4], SR, cap))                                      # warm-up
    ours, dt = timed(lambda: dict(M.evaluate_pairs(items, SR, cap)))
    res["evaluate_pairs_device"] = {"seconds": round(dt, 3), "audio_s_per_s": round(audio_s / dt, 1)}
    print(json.dumps(res["evaluate_pairs_device"]), file=sys.stderr)

    res["kernel_one_pack"] = kernel_times(dev_clips, cap, args.reps)
    print(json.dumps(res["kernel_one_pack"]), file=sys.stderr)

    reference_way(dev_clips[:2], dev)                                               # warm-up (cuFFT plans)
    ref_scores, dt = timed(lambda: reference_way(dev_clips, dev))
    res["reference_way_torch_stft_fp32"] = {"seconds": round(dt, 3), "audio_s_per_s": round(audio_s / dt, 1)}
    res["max_abs_ms_stft_diff_vs_reference_way"] = max(abs(ours[k]["ms_stft"] - ref_scores[k]) for k in ref_scores)
    res["max_rel_ms_stft_diff_vs_reference_way"] = max(abs(ours[k]["ms_stft"] - ref_scores[k]) / abs(ref_scores[k])
                                                       for k in ref_scores)
    print(json.dumps(res["reference_way_torch_stft_fp32"]), file=sys.stderr)

    nd = min(args.disk_clips, args.clips)
    with tempfile.TemporaryDirectory() as tmp:
        rd, dd = os.path.join(tmp, "ref"), os.path.join(tmp, "deg")
        os.makedirs(rd)
        os.makedirs(dd)
        for k, r, d in clips[:nd]:
            offline.write_wav(os.path.join(rd, k + ".wav"), r, SR)
            offline.write_wav(os.path.join(dd, k + ".wav"), d, SR)
        disk_s = sum(r.numel() for _, r, _ in clips[:nd]) / SR

        def from_disk():
            def gen():
                for name, rp, dp in offline.pair_files(rd, dd):
                    r, rsr = offline.read_wav(rp)
                    d, dsr = offline.read_wav(dp)
                    yield name, r, rsr, d, dsr
            return dict(M.evaluate_pairs(gen(), SR, cap))
        _, dt = timed(from_disk)
    res["evaluate_pairs_wav_files"] = {"clips": nd, "audio_seconds": round(disk_s, 1), "seconds": round(dt, 3),
                                       "audio_s_per_s": round(disk_s / dt, 1)}
    summary = M.corpus_summary(ours)
    res["corpus"] = {k: summary[k] for k in ("ms_stft", "sisnr", "stft_skipped", "sisnr_skipped")}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
