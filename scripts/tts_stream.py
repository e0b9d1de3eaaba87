"""Streamed TTS (InferenceImp.stream_many, serve.TTSEngine) at 7B shapes with random init in bf16, the synthetic Mimi
weights and the ragged corpus of scripts/tts_batch.py.  Prints one JSON line:

  * tokens/s (9 per generated frame) of generate_many alone, of generate_many followed by a decode of every utterance
    after generation (MimiCodec.decode_many), and of stream_many, alternated at each capacity, with whether the three
    gave the same codes;
  * a seeded arrival trace into TTSEngine: the time from submit to an utterance's first chunk (p50 / p99), and the
    per-utterance chunk cadence (time between consecutive chunks, p50 / p99) against the 80 ms a chunk lasts;
  * the card's name and power limit, read in the same run.

usage: python scripts/tts_stream.py [--utts 64] [--capacities 32,48] [--trace-utts 48] [--trace-gmax 250] [--out FILE]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from rstnet_b200.codec import MimiCodec   # noqa: E402
from rstnet_b200.infer import InferenceImp   # noqa: E402
from rstnet_b200.serve import TTSEngine   # noqa: E402
from specs import mimi_spec as S   # noqa: E402
from tts_batch import TEXT_EMPTY, corpus, gpt7b   # noqa: E402


def gen_only(imp, codec, items, cap):
    return {u: c.cpu() for u, c in imp.generate_many(items, cap)}


def gen_then_decode(imp, codec, items, cap):
    """generate_many, then every utterance's codes decoded in one continuous batch (MimiCodec.decode_many, capacity 64).
    offline.write_codes_wav's per-length decode keeps one codec plan per distinct length, which does not fit beside the
    7B scope for a corpus of many lengths."""
    codes = {u: c.cpu() for u, c in imp.generate_many(items, cap)}
    for _ in codec.decode_many(((u, c.clamp(max=2047)) for u, c in codes.items() if c.shape[-1]), 64):
        pass
    return codes


def stream(imp, codec, items, cap):
    return {c.utt_id: c.codes for c in imp.stream_many(items, cap, codec) if c.codes is not None}


def pct(x, q):
    return float(np.percentile(np.asarray(x), q)) if len(x) else None


def trace(imp, codec, items, cap, rate_hz, seed):
    """Poisson arrivals (rate_hz requests/s) into a TTSEngine stepped as fast as it goes."""
    rng = np.random.default_rng(seed)
    arrivals = np.cumsum(rng.exponential(1.0 / rate_hz, len(items)))
    submitted, first, last_chunk, gaps = {}, {}, {}, []
    with TTSEngine(imp, codec, cap) as eng:
        t0 = time.perf_counter()
        k = 0
        while k < len(items) or eng.pending or eng.active:
            now = time.perf_counter() - t0
            while k < len(items) and arrivals[k] <= now:
                eng.submit(*items[k])
                submitted[items[k][0]] = time.perf_counter()
                k += 1
            if not (eng.pending or eng.active):
                time.sleep(max(0.0, arrivals[k] - now))
                continue
            out = eng.step()
            t = time.perf_counter()
            for c in out:
                if c.utt_id not in first:
                    first[c.utt_id] = t - submitted[c.utt_id]
                elif c.pcm.numel():
                    gaps.append(t - last_chunk[c.utt_id])
                last_chunk[c.utt_id] = t
        wall = time.perf_counter() - t0
    ms = lambda v: None if v is None else 1e3 * v
    return {"capacity": cap, "requests": len(items), "arrival_rate_per_s": rate_hz, "seconds": wall,
            "first_chunk_ms_p50": ms(pct(list(first.values()), 50)), "first_chunk_ms_p99": ms(pct(list(first.values()), 99)),
            "chunk_gap_ms_p50": ms(pct(gaps, 50)), "chunk_gap_ms_p99": ms(pct(gaps, 99)),
            "chunk_gaps_over_80ms_share": float(np.mean(np.asarray(gaps) > 0.08)) if gaps else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--capacities", default="32,48")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--trace-utts", type=int, default=48)
    ap.add_argument("--trace-gmax", type=int, default=250, help="trace requests generate at most this many frames")
    ap.add_argument("--trace-rate", type=float, default=4.0, help="trace arrivals per second")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tts_stream.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    res = {"model": "7B shapes, random init, bf16, context 2048; Mimi with the synthetic weights",
           "gpu": torch.cuda.get_device_name(dev)}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        res["power_limit"] = f"unknown ({e})"
    m = gpt7b(dev)
    imp = InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")
    codec = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    codec.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
    codec = codec.to(dev).eval()
    items = corpus(args.utts, args.seed)
    frames = sum(int((s[0] == TEXT_EMPTY).sum()) for _, s in items)
    res.update(utterances=len(items), generated_frames=frames, runs={})
    warm = [(u, s[:, :s.shape[1] - int((s[0] == TEXT_EMPTY).sum()) + 8]) for u, s in items]
    modes = {"generate_many": gen_only, "generate_many+decode": gen_then_decode, "stream_many": stream}
    for cap in [int(c) for c in args.capacities.split(",")]:
        digests, row = set(), {}
        for name, fn in modes.items():
            fn(imp, codec, warm[:cap + 4], cap)
        for name, fn in modes.items():       # alternated: every mode once per capacity, back to back
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(imp, codec, items, cap)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            digests.add(hashlib.sha256(b"".join(out[u].numpy().tobytes() for u, _ in items)).hexdigest())
            row[name] = {"seconds": wall, "tokens_per_s": 9 * frames / wall}
            del out
            torch.cuda.empty_cache()
        row["stream_cost_vs_generate_many"] = row["stream_many"]["seconds"] / row["generate_many"]["seconds"] - 1
        row["codes_identical"] = len(digests) == 1
        res["runs"][str(cap)] = row
        print(json.dumps({cap: row}), file=sys.stderr, flush=True)
    g = torch.Generator().manual_seed(args.seed + 1)
    titems = []
    for u, s in corpus(args.trace_utts, args.seed + 1):
        P = s.shape[1] - int((s[0] == TEXT_EMPTY).sum())
        G = int(torch.randint(50, args.trace_gmax + 1, (1,), generator=g))
        titems.append((u, s[:, :P + G]))
    trace(imp, codec, [(f"w{u}", s) for u, s in titems[:8]], 32, 1000.0, args.seed)      # warm-up
    res["trace"] = trace(imp, codec, titems, 32, args.trace_rate, args.seed)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
