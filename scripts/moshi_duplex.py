"""Concurrent duplex sessions of the Moshi 7B model (moshi/models/loaders.py `_lm_kwargs`: dim 4096, 32 layers,
context 3000, text_card 32000, card 2048, depformer 6 x 1024 with weights per step) on one GPU, through
`serve.FrameScheduler` + `serve.MoshiDuplexEngine` (Mimi encode -> LMGen.step -> Mimi decode per 80 ms tick).

Seeded random bf16 LM weights and the specs/mimi_spec.py codec weights; every KV ring is filled to `context` (the rows
are fast-forwarded to step `context`, the steady state of a long session).  LMGen samples with its defaults (top-k 250 /
25, the reference server's settings).  Reports:

  tick    p50 / p99 of a scheduler tick at B = 8, 16, 32 and at the largest B whose KV rings fit in the free memory
          (about 1.57 GB per stream at context 3000);
  frame   device time of one LMGen.step alone (events around graph replays), and of the previous form of the step -- the
          delay cache as eager torch ops around `forward_step`, restated below -- alternated with it;
  launch  host-side launches per step of both forms (torch.profiler: kernel launches, copies, memsets, graph launches).

Prints the card and its power limit, then everything as one JSON line (also written to --out FILE).

    python scripts/moshi_duplex.py [--batches 8,16,32,max] [--ticks 60] [--out FILE]
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
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from rstnet_b200.codec import MimiCodec  # noqa: E402
from rstnet_b200.moshi import LMGen, LMModel  # noqa: E402
from rstnet_b200.serve import FRAME_SAMPLES, FrameScheduler, MoshiDuplexEngine  # noqa: E402
from specs import mimi_spec as S  # noqa: E402

DEV, BF = "cuda", torch.bfloat16
MOSHI_7B = dict(dim=4096, text_card=32000, existing_text_padding_id=3, n_q=16, dep_q=8, card=2048, num_heads=32, num_layers=32,
                hidden_scale=4.125, causal=True, layer_scale=None, context=3000, max_period=10000, gating="silu",
                norm="rms_norm_f32", positional_embedding="rope", depformer_dim=1024, depformer_dim_feedforward=int(4.125 * 1024),
                depformer_num_heads=16, depformer_num_layers=6, depformer_causal=True, depformer_layer_scale=None,
                depformer_multi_linear=True, depformer_context=8, depformer_max_period=10000, depformer_gating="silu",
                depformer_pos_emb="none", depformer_weights_per_step=True,
                delays=[0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1])


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    name, power, clock = ([s.strip() for s in line.split(",")] + ["?", "?", "?"])[:3]
    return {"name": name or torch.cuda.get_device_name(0), "power_limit": power, "max_sm_clock": clock}


def kv_bytes_per_stream(lm: LMModel) -> int:
    c = lm.config
    return c.n_layer * 2 * c.n_head * c.context * c.head_size * 2


def fast_forward(gen: LMGen) -> None:
    """Every row at step `context`: full KV rings, past the warm-up, a cache of valid ids."""
    st, ms, ctx = gen._st, gen._st.lm, gen.lm_model.context
    ms.offset.fill_(ctx)
    ms.pos_host[:] = ctx
    st.cache.fill_(0)
    st.off.fill_(ctx)
    st.off_host[:] = ctx
    st.valid.fill_(1)


def parent_step(gen: LMGen, cache: torch.Tensor, offset: int, input_tokens: torch.Tensor):
    """The previous LMGen.step: the delay cache as eager torch ops around one `forward_step` graph replay."""
    lm = gen.lm_model
    CT = cache.shape[2]
    for q in range(input_tokens.shape[1]):
        k = lm.dep_q + 1 + q
        wp = (offset + lm.delays[k]) % CT
        cache[:, k, wp:wp + 1] = input_tokens[:, q]
    position = offset % CT
    for k, delay in enumerate(lm.delays):
        if offset <= delay:
            cache[:, k, position] = lm.text_initial_token_id if k == 0 else lm.initial_token_id
    input_ = cache[:, :, position:position + 1]
    toks = lm._st().forward_step(input_, gen.use_sampling, gen.temp_text, gen.top_k_text, gen.temp, gen.top_k, lm.card, True)
    offset += 1
    position = offset % CT
    cache[:, 0, position] = toks[:, 0]
    cache[:, 1:lm.dep_q + 1, position] = toks[:, 1:]
    index = ((offset - gen.max_delay + gen.delays_cuda[:lm.dep_q + 1]) % CT).view(1, -1, 1).expand(cache.shape[0], -1, 1)
    return cache.gather(dim=2, index=index), offset


def count_launches(fn) -> dict:
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    out = {"kernel": sum(n.startswith("cudaLaunchKernel") for n in names),
           "memcpy": sum(n.startswith("cudaMemcpy") for n in names),
           "memset": sum(n.startswith("cudaMemset") for n in names),
           "graph": sum(n == "cudaGraphLaunch" for n in names)}
    out["total"] = sum(out.values())
    return out


def frame_part(lm: LMModel, B: int, reps: int) -> dict:
    """LMGen.step alone vs the previous form, same scope, alternated in blocks of `reps` steps."""
    gen = LMGen(lm)
    gen.streaming_forever(B)
    fast_forward(gen)
    codes = torch.randint(0, lm.card, (B, lm.n_q - lm.dep_q, 1), device=DEV)
    cache = torch.zeros(B, lm.num_codebooks, gen.max_delay + 2, dtype=torch.long, device=DEV)
    off = [lm.context]

    def new():
        gen.step(codes)

    def old():
        _, off[0] = parent_step(gen, cache, off[0], codes)

    for f in (new, old):
        for _ in range(3):
            f()
    res = {"launches_new": count_launches(new), "launches_old": count_launches(old)}
    ev = lambda: torch.cuda.Event(enable_timing=True)
    times = {"new": [], "old": []}
    host = {"new": [], "old": []}
    for _ in range(5):
        for name, f in (("new", new), ("old", old)):
            torch.cuda.synchronize()
            a, b = ev(), ev()
            t0 = time.perf_counter()
            a.record()
            for _ in range(reps):
                f()
            b.record()
            torch.cuda.synchronize()
            host[name].append(1e3 * (time.perf_counter() - t0) / reps)
            times[name].append(a.elapsed_time(b) / reps)
    for name in ("new", "old"):
        res[f"frame_ms_{name}"] = {"median": float(np.median(times[name])), "min": float(np.min(times[name])),
                                   "max": float(np.max(times[name])), "host_ms_median": float(np.median(host[name]))}
    gen._st = None
    lm._state = None
    return res


def tick_part(lm: LMModel, codec: MimiCodec, B: int, ticks: int) -> dict:
    gen = LMGen(lm)
    eng = MoshiDuplexEngine(codec, gen, B)
    sch = FrameScheduler(eng, B)
    for s in range(B):
        sch.admit(s)
    fast_forward(gen)
    x = S.synthetic_audio(B, FRAME_SAMPLES * 8, seed=3)[:, 0]
    lat = []
    for t in range(ticks + 5):
        for s in range(B):
            i = t % 8
            sch.push(s, x[s, i * FRAME_SAMPLES:(i + 1) * FRAME_SAMPLES])
        t0 = time.perf_counter()
        out = sch.tick()
        dt = 1e3 * (time.perf_counter() - t0)
        if t >= 5:
            lat.append(dt)
    assert len(out) == B and all(p is not None and bool(torch.isfinite(p).all()) for _, p in out.values())
    res = {"B": B, "tick_ms_p50": float(np.percentile(lat, 50)), "tick_ms_p99": float(np.percentile(lat, 99)),
           "tick_ms_max": float(np.max(lat)), "ticks": len(lat)}
    codec._stream_state = None
    gen._st = None
    lm._state = None
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="8,16,32,max")
    ap.add_argument("--ticks", type=int, default=60)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moshi_duplex.py measures on a CUDA device; none is visible")
    res = {"card": card(), "model": "moshi-7b shapes (loaders.py _lm_kwargs), random bf16 weights"}
    print(json.dumps(res["card"]), flush=True)
    torch.manual_seed(0)
    lm = LMModel(**MOSHI_7B, device=DEV, dtype=BF).eval()
    codec = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    codec.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
    codec = codec.to(DEV).eval()
    per = kv_bytes_per_stream(lm)
    res["weights_gb"] = sum(p.numel() * p.element_size() for p in lm.parameters()) / 1e9
    res["kv_gb_per_stream"] = per / 1e9
    res["frame"] = {}
    for B in (8, 32):
        res["frame"][B] = frame_part(lm, B, a.reps)
        gc.collect(); torch.cuda.empty_cache()
        print(json.dumps({"frame": {B: res["frame"][B]}}), flush=True)
    res["tick"] = []
    for b in a.batches.split(","):
        if b == "max":
            gc.collect(); torch.cuda.empty_cache()
            free, _ = torch.cuda.mem_get_info()
            B = int((free - 3e9) // per)                        # 3 GB for the codec scope, activations and graphs
            res["max_B_estimate"] = B
        else:
            B = int(b)
        while B > 0:
            try:
                r = tick_part(lm, codec, B, a.ticks)
                break
            except torch.cuda.OutOfMemoryError:
                codec._stream_state = None; lm._state = None
                gc.collect(); torch.cuda.empty_cache()
                res.setdefault("oom", []).append(B)
                B -= 1
        res["tick"].append(r)
        print(json.dumps(r), flush=True)
        gc.collect(); torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
