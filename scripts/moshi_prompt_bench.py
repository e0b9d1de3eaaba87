"""Prompted Moshi generation at Moshi 7B shapes (moshi/models/loaders.py `_lm_kwargs`, seeded random bf16 weights) on one
GPU.  Prints the card and its power limit, then one JSON line (also written to --out FILE).

  (a) admission   a prompted session (P = 125 / 375 / 750 frames) admitted through FrameScheduler into a paged
                  MoshiDuplexEngine whose other B - 1 = 31 rows are live sessions: the wall time from `admit` to the
                  session's first output frame, and the tick times of the live sessions until then (each tick ends in a
                  device synchronise).  For comparison, the median tick of the same scope without an admission, times P:
                  what feeding the prompt one frame per tick would take.
  (b) generation  moshi.generate_many over a seeded ragged corpus of 64 dialogues (P uniform in 0..500, L - P in
                  100..1000), paged, at capacity 32 and 48: frames/s (live rows summed over steps, over wall time that ends
                  in a synchronise), and the same corpus with P = 0.  At capacity 32 a second run synchronises around each
                  prefill call to give the prefill's share of the wall time.

    python scripts/moshi_prompt_bench.py [--out FILE] [--quick]
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

from rstnet_b200.codec import MimiCodec  # noqa: E402
from rstnet_b200.lm import kv_pages_for_budget  # noqa: E402
from rstnet_b200.moshi import LMGen, LMModel, generate_many, prompt_from_aligned  # noqa: E402
from rstnet_b200.serve import FRAME_SAMPLES, FrameScheduler, MoshiDuplexEngine  # noqa: E402
from scripts.moshi_duplex import MOSHI_7B, card  # noqa: E402
from specs import mimi_spec as S  # noqa: E402

DEV, BF = "cuda", torch.bfloat16


def _seq(lm, L, seed):
    g = torch.Generator().manual_seed(seed)
    s = torch.randint(0, lm.card, (lm.num_codebooks, L), generator=g)
    s[0] = torch.randint(0, lm.text_card, (L,), generator=g)
    return s


def admission(lm, codec, B, Ps, warm_ticks):
    lm_gen = LMGen(lm)
    pool = kv_pages_for_budget(lm.config, 24.0)
    eng = MoshiDuplexEngine(codec, lm_gen, B, kv_pages=pool)
    sch = FrameScheduler(eng, B)
    pcm = S.synthetic_audio(1, FRAME_SAMPLES, seed=3)[0, 0]
    for i in range(B - 1):
        sch.admit(f"live{i}", seed=i)

    def tick():
        for s in sch.sessions():
            sch.push(s, pcm)
        t0 = time.perf_counter()
        out = sch.tick()
        return out, 1e3 * (time.perf_counter() - t0)
    for _ in range(warm_ticks):
        tick()
    base = [tick()[1] for _ in range(warm_ticks)]
    res = {"tick_ms_p50_no_admission": float(np.percentile(base, 50)), "cases": []}
    for j, P in enumerate(Ps):
        for rep in range(2):                     # the first admission of a size warms its chunk shapes
            prompt = prompt_from_aligned(_seq(lm, P, 7 + j), P, lm.delays, lm.dep_q)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            sch.admit("p", seed=99, prompt=prompt)
            ticks = []
            while True:
                out, ms = tick()
                ticks.append(ms)
                if "p" in out:
                    break
            first = 1e3 * (time.perf_counter() - t0)
            sch.release("p")
        res["cases"].append({"P": P, "admit_to_first_frame_ms": first, "ticks": len(ticks),
                             "live_tick_ms_p50": float(np.percentile(ticks, 50)),
                             "live_tick_ms_p99": float(np.percentile(ticks, 99)),
                             "P_ticks_ms": P * res["tick_ms_p50_no_admission"]})
        print(json.dumps(res["cases"][-1]), flush=True)
    codec._stream_state = None
    lm._state = None                  # free the engine's KV pool before the generation runs
    del sch, eng, lm_gen
    gc.collect()
    torch.cuda.empty_cache()
    return res


def corpus(lm, n, zero_prompt):
    g = np.random.default_rng(5)
    items = []
    for i in range(n):
        P, G = int(g.integers(0, 501)), int(g.integers(100, 1001))
        items.append((f"d{i}", _seq(lm, P + G, 100 + i), 0 if zero_prompt else P))
    return items


def generation(lm, capacity, items, time_prefill=False):
    gen = LMGen(lm)
    pool = kv_pages_for_budget(lm.config, 36.0)
    prefill = [0.0]
    if time_prefill:
        inner = gen.prefill_streams

        def timed(prompts):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            inner(prompts)
            torch.cuda.synchronize()
            prefill[0] += time.perf_counter() - t0
        gen.prefill_streams = timed
    stats = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = sum(o.shape[1] for _, o in generate_many(gen, items, capacity, seeds={u: i for i, (u, _, _) in enumerate(items)},
                                                  kv_pages=pool, stats=stats))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    out = {"capacity": capacity, "frames_per_s": n / dt, "seconds": dt, "steps": stats["frames"],
           "prefill_frames": stats["prefill_rows"]}
    if time_prefill:
        out["prefill_share"] = prefill[0] / dt
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true", help="fewer items and ticks (a rehearsal, not a measurement)")
    args = ap.parse_args()
    info = card()
    print(json.dumps({"card": info}), flush=True)
    lm = LMModel(**MOSHI_7B, device=DEV, dtype=BF).eval()
    codec = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    codec.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
    codec = codec.to(DEV).eval()
    res = {"card": info, "model": "Moshi 7B shapes, random bf16 weights"}
    res["admission"] = admission(lm, codec, 32, [125, 375, 750], 5 if args.quick else 30)
    n = 8 if args.quick else 64
    prompted, zero = corpus(lm, n, False), corpus(lm, n, True)
    generation(lm, 32, prompted[:4])                                     # warm-up of the shapes
    res["generation"] = []
    for cap in (32, 48):
        res["generation"].append({"prompted": generation(lm, cap, prompted), "P0": generation(lm, cap, zero)})
    res["generation_prefill_timed"] = generation(lm, 32, prompted, time_prefill=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
