"""Forced tokens during Moshi generation at Moshi 7B shapes (seeded random bf16 weights) on one GPU.  Prints the card and
its power limit, then one JSON line (also written to --out FILE).

  (a) frame time  LMGen.step at B = 32 on a paged scope, three graphs alternated step by step within one scope: the
                  plain frame, the forced frame with nothing forced (every id -1) and the forced frame with the audio
                  codebooks forced (text sampled).  Each step's device time between CUDA events recorded between the
                  steps (the table copy before a forced replay included); per graph the median and mean, and the mean
                  difference to the plain steps around it, interpolated to its position (the frame time grows with the
                  KV length, one position per step).
  (b) throughput  moshi.generate_many over the corpus of scripts/moshi_prompt_bench.py (64 dialogues, P uniform in 0..500,
                  L - P in 100..1000), paged, capacity 32: no forcing against every item's audio forced at every frame
                  (`offline continue --force audio`), alternated; live-row frames/s over wall time ending in a synchronise.

    python scripts/forced_gen_bench.py [--out FILE] [--quick]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from rstnet_b200.lm import kv_pages_for_budget  # noqa: E402
from rstnet_b200.moshi import LMGen, LMModel, generate_many  # noqa: E402
from scripts.moshi_duplex import MOSHI_7B, card  # noqa: E402
from scripts.moshi_prompt_bench import corpus  # noqa: E402

DEV, BF = "cuda", torch.bfloat16


def frame_times(lm, B, frames):
    """`frames` steps of each graph, interleaved step by step (plain, forced with nothing forced, audio forced, ...) so
    that the three see the same KV lengths; each step timed by the CUDA events recorded between the steps"""
    gen = LMGen(lm)
    K, dq = lm.num_codebooks, lm.dep_q
    g = torch.Generator().manual_seed(1)
    x = torch.randint(0, lm.card, (B, K - dq - 1, 1), generator=g).to(DEV)
    none = torch.full((B, dq + 1, 1), -1, dtype=torch.int64, device=DEV)
    audio = torch.randint(0, lm.card, (B, dq + 1, 1), generator=g).to(DEV)
    audio[:, 0] = -1
    modes = {"plain": None, "forced_nothing": none, "forced_audio": audio}
    warm = 3 * len(modes)                            # captures and warms the three graphs
    n = warm + frames * len(modes)
    with gen.streaming(B, kv_pages=kv_pages_for_budget(lm.config, 24.0)), torch.no_grad():
        gen.reserve_kv(list(range(B)), n)
        gen.set_stream_sampling(list(range(B)), None, 7)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
        forces = list(modes.values())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            ev[i].record()
            gen.step(x, force=forces[i % len(modes)])
        ev[n].record()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    ms = np.array([ev[i].elapsed_time(ev[i + 1]) for i in range(warm, n)]).reshape(frames, len(modes))
    out = {"B": B, "frames_per_graph": frames, "wall_s": wall}
    for j, name in enumerate(modes):
        out[name] = {"device_ms_median": float(np.median(ms[:, j])), "device_ms_mean": float(ms[:, j].mean())}
        if j:
            # against the plain steps around it, interpolated to its position (the frame time grows with the KV length)
            plain = ms[:-1, 0] + (ms[1:, 0] - ms[:-1, 0]) * j / len(modes)
            d = ms[:-1, j] - plain
            out[name]["vs_plain_ms_mean"] = float(d.mean())
            out[name]["vs_plain_ms_median"] = float(np.median(d))
            out[name]["vs_plain_frac"] = float(d.mean() / plain.mean())
    print(json.dumps(out), flush=True)
    lm._state = None                  # free the scope's KV pool before the generation runs
    gc.collect()
    torch.cuda.empty_cache()
    return out


def throughput(lm, items, capacity, force_audio):
    gen = LMGen(lm)
    dq = lm.dep_q
    masks = None
    if force_audio:
        masks = {u: (torch.arange(dq + 1)[:, None] > 0).expand(dq + 1, s.shape[1]).clone() for u, s, _ in items}
    stats = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = sum(o.shape[1] for _, o in generate_many(gen, items, capacity, seeds={u: i for i, (u, _, _) in enumerate(items)},
                                                  kv_pages=kv_pages_for_budget(lm.config, 36.0), stats=stats, force=masks))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    out = {"capacity": capacity, "force": "audio" if force_audio else None, "frames_per_s": n / dt, "seconds": dt,
           "steps": stats["frames"]}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="fewer frames and items (a rehearsal, not a measurement)")
    args = ap.parse_args()
    info = card()
    print(json.dumps({"card": info}), flush=True)
    lm = LMModel(**MOSHI_7B, device=DEV, dtype=BF).eval()
    res = {"card": info, "model": "Moshi 7B shapes, random bf16 weights"}
    res["frame"] = frame_times(lm, 32, 20 if args.quick else 300)
    items = corpus(lm, 8 if args.quick else 64, False)
    throughput(lm, items[:4], 32, False)                 # warm-up of the shapes
    throughput(lm, items[:4], 32, True)
    res["throughput"] = [throughput(lm, items, 32, fa) for fa in (False, True, False, True)]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
