"""Resampling on one GPU:

  (a) kernel   rstnet_resample_f32 on 256 rows x 10 s for every rate pair of tests/resample_oracle.PAIRS: ms per launch
               (CUDA events over >= 20 launches after warm-up), algorithmic bytes 4 * (rows * L_in + rows * L_out), GB/s
               and share of the H100 SXM data sheet's 3.35 TB/s; beside it, torchaudio's arithmetic on the same GPU
               (pad + F.conv1d with the full table, stride o + transpose / truncate);
  (b) offline  256 clips x 10 s through offline.tokenize_utterances at 24 kHz and at 16 kHz;
  (c) duplex   DuplexEngine tick p50 / p99 at B = 48 for 24 / 16 / 48 kHz clients, alternated in one process, with
               bench.py cfg 5's setup (7B random init, LM KV rings and codec rings full).

Prints the card and its power limit (read in the same call) and every result as one JSON line; --out FILE also writes it.

    python scripts/resample_bench.py [--parts kernel,offline,duplex] [--out FILE]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import resample_oracle as R  # noqa: E402
from rstnet_b200 import audio  # noqa: E402

DEV = "cuda"
HBM_BYTES_PER_S = 3.35e12
FP32_FLOP_PER_S = 67e12


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    name, power, clock = ([s.strip() for s in line.split(",")] + ["?", "?", "?"])[:3]
    return {"name": name or torch.cuda.get_device_name(0), "power_limit": power, "max_sm_clock": clock}


def time_events(fn, reps: int = 20, warmup: int = 3) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def kernel_part(rows: int = 256, seconds: float = 10.0):
    out = []
    for orig, new in R.PAIRS:
        rs = audio.Resample(orig, new)
        t = rs.table
        L = int(seconds * orig)
        x = torch.randn(rows, L, device=DEV) * 0.3
        L_out = rs.output_length(L)
        ms = time_events(lambda: rs(x), reps=30)
        nbytes = 4.0 * (rows * L + rows * L_out)
        runs = (t.taps != 0).sum(1).double()
        flops_trim = 2.0 * rows * t.S * L_out                  # FMAs the kernel issues (padded taps included)
        flops_full = 2.0 * rows * t.K * L_out                  # the full table, as conv1d computes it
        t_mem, t_fma = nbytes / HBM_BYTES_PER_S, flops_trim / FP32_FLOP_PER_S
        kern = R.sinc_kernel(orig, new)[0].to(DEV)
        ms_conv = time_events(lambda: R.apply_kernel(x, orig, new, kern, t.width), reps=20)
        out.append({"pair": f"{orig}->{new}", "o": t.o, "n": t.n, "S": t.S, "K": t.K, "mean_run": float(runs.mean()),
                    "rows": rows, "L_in": L, "L_out": L_out, "ms": ms, "bytes": nbytes, "GB_per_s": nbytes / ms * 1e-6,
                    "bound": "HBM" if t_mem >= t_fma else "FP32 FMA",
                    "share_of_bound": max(t_mem, t_fma) * 1e3 / ms,
                    "gflop_trimmed": flops_trim * 1e-9, "gflop_full": flops_full * 1e-9,
                    "torch_conv1d_full_table_ms": ms_conv, "speedup_vs_conv1d": ms_conv / ms})
        del x, kern
        torch.cuda.empty_cache()
    return out


def offline_part(clips: int = 256, seconds: float = 10.0):
    from oracle import mimi_spec as S
    from rstnet_b200 import offline
    from rstnet_b200.codec import MimiCodec
    m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
    m = m.to(DEV).eval()
    res = {}
    base = S.synthetic_audio(8, int(seconds * 24000), seed=3)[:, 0]
    for rate in (24000, 16000, 24000, 16000):                 # alternated; the second of each is reported
        L = int(seconds * rate)
        wav = torch.nn.functional.interpolate(base[:, None], size=L, mode="linear")[:, 0] if rate != 24000 else base
        items = [(f"u{i}", wav[i % 8], rate) for i in range(clips)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        toks = offline.tokenize_utterances(m, items, batch_size=32)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        rs_ms = 0.0
        if rate != 24000:
            rs = audio.Resample(rate, 24000)
            x = torch.stack([w for _, w, _ in items]).to(DEV)
            rs_ms = time_events(lambda: rs(x), reps=20)
        res[str(rate)] = {"clips": clips, "seconds_each": seconds, "wall_s": dt, "audio_s_per_wall_s": clips * seconds / dt,
                          "resample_ms": rs_ms, "resample_share": rs_ms * 1e-3 / dt, "frames": int(sum(v.shape[1] for v in toks.values()))}
    del m
    gc.collect()
    torch.cuda.empty_cache()
    return res


def duplex_part(B: int = 48, ticks: int = 40):
    import bench
    from oracle import mimi_spec as S
    from rstnet_b200.serve import DuplexEngine, FrameScheduler
    codec = bench._mimi(DEV, S)
    lm = bench._gpt7b(DEV, context=2048)
    src = S.synthetic_audio(8, 1920 * 8, seed=12)[:, 0]
    lat = {r: [] for r in (24000, 16000, 48000)}
    for rnd in range(2):                                       # 24 / 16 / 48 kHz alternated, twice
        for rate in lat:
            F = rate * 2 // 25
            frames = torch.nn.functional.interpolate(src[:, None], size=F * 8, mode="linear")[:, 0] if rate != 24000 else src
            eng = DuplexEngine(codec, lm, B, sample_rate=rate)
            sch = FrameScheduler(eng, B)
            for s in range(B):
                sch.admit(s)
            for tick in range(ticks // 2 + 6):
                if tick == 3:
                    st = lm._state
                    for kv in st.kv:
                        kv.normal_()
                    st.offset.fill_(2048 + 100); st.pos_host[:] = 2048 + 100
                    for plan in list(codec._stream_state.enc.values()) + list(codec._stream_state.dec.values()):
                        plan.offset.fill_(1000)
                for s in range(B):
                    sch.push(s, frames[s % 8, (tick % 8) * F:(tick % 8 + 1) * F])
                assert len(sch.tick()) == B
            lat[rate] += eng.latencies_ms[6:]
            lm._state = None
            codec._stream_state = None
            eng = sch = st = plan = kv = None
            gc.collect()
            torch.cuda.empty_cache()
    res = {}
    for rate, v in lat.items():
        v = sorted(v)
        p = lambda q: v[min(len(v) - 1, int(q * len(v)))]
        res[str(rate)] = {"streams": B, "ticks": len(v), "tick_ms_p50": p(0.5), "tick_ms_p99": p(0.99)}
    return res


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--parts", default="kernel,offline,duplex")
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("resample_bench.py needs a CUDA device")
    parts = args.parts.split(",")
    res = {"card": card(), "hbm_peak_TB_per_s": HBM_BYTES_PER_S * 1e-12}
    if "kernel" in parts:
        res["kernel"] = kernel_part()
    if "offline" in parts:
        res["offline"] = offline_part()
    if "duplex" in parts:
        res["duplex"] = duplex_part()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
