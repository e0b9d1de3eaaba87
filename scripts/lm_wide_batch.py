"""Decode scopes of up to 256 streams on one GPU, measured at the widths of a Llama-3.2-3B-shaped LM (GQA 24 / 8,
n_embd 3072, intermediate 8192) with the recipe's depth transformer:

  (a) gemm    the weight-streaming GEMM at M = 128, at M = 256 and as two M = 128 launches: time per call and achieved
              weight bandwidth (weight bytes / time) for QKV, the interleaved fc_1/fc_2 (fc12), proj, down and lm_head;
              plus, at M = 256, every split count the plan can take for the split-K shapes of the LM;
  (b) decode  ms per forward_step frame (temporal step + text sampling + 8 depth steps) at B = 128, 192, 256 with every
              KV ring full (2048-key window, wrapped);
  (c) duplex  tick p50 / p99 through serve.DuplexEngine (Mimi encode -> LM frame -> Mimi decode) at 128, 192, 256
              streams, and the largest batch whose p99 stays under the 80 ms frame period.

A batch that does not fit in the free memory is recorded as out of memory.  Prints the card and its power limit, then
everything as one JSON line, which --out FILE also writes to FILE.

    python scripts/lm_wide_batch.py [--parts gemm,decode,duplex] [--out FILE]
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

import torch  # noqa: E402

from rstnet_b200.lm import GPT, Config, SkinnyGemm, interleave_gate_rows  # noqa: E402

DEV, BF = "cuda", torch.bfloat16
KV_KEYS = 2048
SPLITS = (1, 2, 3, 4, 6, 8)


def llama32_3b() -> Config:
    return Config(block_size=4096, n_layer=28, n_embd=3072, n_head=24, n_query_groups=8, head_size=128, intermediate_size=8192,
                  rope_base=500000, rope_adjustments={"factor": 32.0, "low_freq_factor": 1.0, "high_freq_factor": 4.0,
                                                      "original_max_seq_len": 8192},
                  padded_vocab_size=152064, audio_card=2050, n_q=8, dep_q=8, codecformer_dim=1024, codecformer_heads=16,
                  codecformer_layers=6, codecformer_dim_feedforward=4224, context=KV_KEYS)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    name, power, clock = ([s.strip() for s in line.split(",")] + ["?", "?", "?"])[:3]
    return {"name": name or torch.cuda.get_device_name(0), "power_limit": power, "max_sm_clock": clock,
            "sms": torch.cuda.get_device_properties(0).multi_processor_count}


def time_graph(fn, reps: int = 20) -> float:
    """ms per call of fn: fn is captured once into a CUDA graph and the graph replayed `reps` times between events."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


# ----------------------------------------------------------------------------------------------------------- (a)
def gemm_part(cfg: Config) -> dict:
    E, I, V = cfg.n_embd, cfg.intermediate_size, cfg.padded_vocab_size
    qkv_n = (cfg.n_head + 2 * cfg.n_query_groups) * cfg.head_size
    D, H = cfg.codecformer_dim, cfg.ff_hidden
    Hp = -(-H // 64) * 64
    g = torch.Generator(device=DEV).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=g).to(BF)
    # name: (N, K, mode) with mode 0 plain, 1 residual + RMSNorm, 3 interleaved SiLU gating -- as lm.py plans them
    shapes = {"qkv": (qkv_n, E, 0), "fc12": (2 * I, E, 3), "proj": (E, cfg.n_head * cfg.head_size, 1), "down": (E, I, 1),
              "lm_head": (V, E, 0)}
    depth = {"depth_in": (D, E, 1), "depth_qkv": (3 * D, D, 0), "depth_out": (D, D, 1), "depth_gin": (2 * Hp, D, 2),
             "depth_gout": (D, Hp, 1), "depth_head": (cfg.audio_card, D, 0)}
    wsmax = max(qkv_n, 2 * I, 4096, 3 * D, 2 * Hp)

    def plans(N, K, mode, M, W, max_splits):
        X = rnd(M, K)
        out = rnd(M, N) if mode != 3 else None
        ws = torch.full((8 * M * wsmax,), float("nan"), dtype=torch.float32, device=DEV) if N <= wsmax else None
        kw = {}
        if mode == 1:
            kw = dict(norm_w=rnd(N), aux=rnd(M, N), eps=1e-5)
        elif mode in (2, 3):
            kw = dict(silu_out=rnd(M, N // 2), interleaved=mode == 3)
        return [SkinnyGemm(X, w, out, out if mode == 1 else None, ws, max_splits=max_splits, **kw) for w in W], ws

    def weights(N, K):
        # enough distinct copies that one pass over them does not fit in L2: every call streams its weight from HBM
        n = max(1, -(-(256 << 20) // (N * K * 2)))
        return [rnd(N, K) for _ in range(n)]

    def splits_ran(ws, M, N):
        if ws is None:
            return 1
        w = ~ws[:8 * M * N].view(8, M * N)[:, :1].isnan()
        return max(1, int(w.all(1).sum()))

    res = {"widths": {}, "split_sweep_m256": {}}
    for name, (N, K, mode) in shapes.items():
        W = weights(N, K)
        wbytes = N * K * 2
        row = {"N": N, "K": K}
        for label, M, launches in (("m128", 128, 1), ("m256", 256, 1), ("two_m128", 128, 2)):
            ps = [plans(N, K, mode, M, W, 8)[0] for _ in range(launches)]
            ms = time_graph(lambda: [p.run() for pl in ps for p in pl]) / len(W)
            row[label] = {"ms": round(ms, 4), "weight_gbs": round(launches * wbytes / ms * 1e-6, 1)}
        row["m256_over_m128"] = round(row["m256"]["ms"] / row["m128"]["ms"], 3)
        row["two_m128_over_m256"] = round(row["two_m128"]["ms"] / row["m256"]["ms"], 3)
        res["widths"][name] = row
        print(f"[gemm] {name:8s} N {N:6d} K {K:5d}  M128 {row['m128']['ms']:.4f} ms ({row['m128']['weight_gbs']} GB/s)  "
              f"M256 {row['m256']['ms']:.4f} ms ({row['m256']['weight_gbs']} GB/s)  2xM128 {row['two_m128']['ms']:.4f} ms", flush=True)
        del W
    for name, (N, K, mode) in {k: v for k, v in {**shapes, **depth}.items() if v[0] <= wsmax and v[2] != 3}.items():
        W = weights(N, K)
        sweep = {}
        for c in SPLITS:
            pl, ws = plans(N, K, mode, 256, W, c)
            pl[0].run()
            torch.cuda.synchronize()
            ran = splits_ran(ws, 256, N)
            if str(ran) in sweep:
                continue
            ms = time_graph(lambda: [p.run() for p in pl]) / len(W)
            sweep[str(ran)] = round(ms, 4)
        default = {}
        for M in (128, 256):
            pl, ws = plans(N, K, mode, M, W, 8)
            pl[0].run()
            torch.cuda.synchronize()
            default[f"m{M}"] = splits_ran(ws, M, N)
        best = min(sweep, key=sweep.get)
        res["split_sweep_m256"][name] = {"N": N, "K": K, "mode": mode, "ms_by_splits": sweep, "best": int(best),
                                         "chosen_m256": default["m256"], "chosen_m128": default["m128"]}
        print(f"[split] {name:10s} N {N:5d} K {K:5d} M256 ms by splits {sweep}  best {best}  chosen {default['m256']} "
              f"(M128 chooses {default['m128']})", flush=True)
        del W
    return res


# ----------------------------------------------------------------------------------------------------------- (b)
def fill_rings(lm, B):
    st = lm._state
    for kv in st.kv:
        kv.normal_()
    st.offset.fill_(KV_KEYS + 100)
    st.pos_host[:] = KV_KEYS + 100


def decode_part(lm, batches=(128, 192, 256), steps: int = 20) -> dict:
    res = {}
    for B in batches:
        try:
            lm.streaming_forever(B)
            fill_rings(lm, B)
            seq = torch.randint(0, 2048, (B, 9, 1), device=DEV)
            for _ in range(3):
                lm.forward_step(seq)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                lm.forward_step(seq)
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b) / steps
            res[str(B)] = {"frame_ms": round(ms, 3), "frames_per_s": round(B / ms * 1e3, 1)}
        except torch.cuda.OutOfMemoryError:
            res[str(B)] = {"error": "out of memory"}
        lm._state = None
        gc.collect()
        torch.cuda.empty_cache()
        print(f"[decode] B {B}: {res[str(B)]}", flush=True)
    return res


# ----------------------------------------------------------------------------------------------------------- (c)
def duplex_part(lm, batches=(128, 192, 256), ticks: int = 30) -> dict:
    from rstnet_b200.codec import MimiCodec
    from rstnet_b200.serve import DuplexEngine, FrameScheduler
    from specs import mimi_spec as S
    codec = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    codec.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
    codec = codec.to(DEV).eval()
    audio = S.synthetic_audio(8, 1920 * 8, seed=12)
    res = {"tick_budget_ms": 80.0, "runs": []}
    for B in batches:
        eng = sch = None
        try:
            eng = DuplexEngine(codec, lm, B)
            sch = FrameScheduler(eng, B)
            for s in range(B):
                sch.admit(s)
            for tick in range(ticks + 6):
                if tick == 3:       # long-running sessions: LM rings full (2048 keys, wrapped), codec rings full
                    fill_rings(lm, B)
                    for plan in list(codec._stream_state.enc.values()) + list(codec._stream_state.dec.values()):
                        plan.offset.fill_(1000)
                for s in range(B):
                    sch.push(s, audio[s % 8, 0, (tick % 8) * 1920:(tick % 8 + 1) * 1920])
                assert len(sch.tick()) == B
            lat = sorted(eng.latencies_ms[6:])
            p = lambda q: lat[min(len(lat) - 1, int(q * len(lat)))]
            run = {"streams": B, "tick_ms_p50": round(p(0.5), 2), "tick_ms_p99": round(p(0.99), 2), "realtime": p(0.99) < 80.0}
        except torch.cuda.OutOfMemoryError:
            run = {"streams": B, "error": "out of memory"}
        res["runs"].append(run)
        print(f"[duplex] {run}", flush=True)
        lm._state = None
        codec._stream_state = None
        eng = sch = None
        gc.collect()
        torch.cuda.empty_cache()
    ok = [r["streams"] for r in res["runs"] if r.get("realtime")]
    res["largest_realtime_batch"] = max(ok) if ok else 0
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="gemm,decode,duplex")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    parts = a.parts.split(",")
    cfg = llama32_3b()
    res = {"card": card(), "config": "Llama-3.2-3B shape: 28 x 3072, 24 heads / 8 KV groups, intermediate 8192, vocab 152064, "
                                     "depth 6 x 1024 / 16 heads / ff 4224, KV ring 2048 keys"}
    print(f"card: {res['card']}", flush=True)
    t0 = time.time()
    if "gemm" in parts:
        res["gemm"] = gemm_part(cfg)
        gc.collect()
        torch.cuda.empty_cache()
    if "decode" in parts or "duplex" in parts:
        lm = GPT(cfg, device=DEV, dtype=BF).eval()
        if "decode" in parts:
            res["decode"] = decode_part(lm)
        if "duplex" in parts:
            res["duplex"] = duplex_part(lm)
    res["wall_s"] = round(time.time() - t0, 1)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
