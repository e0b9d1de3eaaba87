#!/usr/bin/env python
"""bench.py — BASELINE.json configs[1]: MimiCodec streaming encode+decode, 256 streams x 10 s of
synthetic 24 kHz audio per GPU (125 frames of 80 ms each, one frame of every stream per launch
sequence), seeded synthetic weights.  Metric: codec frames/s (one frame = 1920 samples encoded to
8 tokens and decoded back); real-time streams = frames/s / 12.5.

  python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]

A "step" = one pass over the whole batch: 125 streaming frames x 256 streams (encode + decode).
`value` is measured with the 10 s inputs already resident in HBM; `e2e` copies every 80 ms chunk
from pinned host memory and reads tokens + waveform back each frame.  Multi-GPU: streams shard
across ranks with no data-path collective (weak scaling); timing = max over ranks.
`--impl reference` times the reference's CPU implementation of the same path (the oracle port, torch
CPU fp32 with all host threads) on a bounded sample.
`--dump-outputs DIR` writes what the last timed step computed (rank 0; collected by an untimed replay of that step, whose
last frame is checked bit for bit against the timed one): DIR/codes.npy, every stream's tokens of the 125
frames [256, 8, 125], and DIR/wav.npy, the decoded 10 s waveforms of a fixed seeded sample of 32 streams [32, 240000]
(stream indices in DIR/wav_streams.npy), all float32.  Inputs are seeded, so two builds can be compared output for output.

Next to the headline (N = 1 only, extra keys, each its own unit of work and outside the headline's timed region):
  steady_state        the same pass with the codec transformers' rings already full (context 250), i.e. what a long-running
                      server sees; the headline's 10 s streams start cold;
  lm_decode           BASELINE configs[2]: one 7B decode step, B = 32, KV ring 2048 (wrapped; 64 streams' rings would not
                      fit next to the weights in 80 GB);
  cfg4_infer          BASELINE configs[3]: Mimi encode -> InferenceImp (prefill + 1000 generated frames) -> Mimi decode, B = 32;
  cfg5_duplex         BASELINE configs[4] on one GPU: batched real-time loop (codec encode -> LM frame -> codec decode per 80 ms
                      tick, rstnet_b200.serve.DuplexEngine), per-tick latency p50 / p99 and the streams that sustain real time;
  gpu_eager_baseline  the reference's eager arithmetic (the oracle port, same ATen calls) on THIS GPU: the same-box
                      comparator BASELINE.md §4 names, for the codec pass and the LM step.
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

STREAMS, SECONDS = 256, 10
FRAMES = int(SECONDS * 12.5)
FRAME = 1920
METRIC, UNIT = "codec_frames_per_s", "frames/s"
WORKLOAD = f"mimi_streaming_encode_decode_B{STREAMS}x{SECONDS}s_24kHz"


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d["bf16_tflops"], "bf16_tflops_sustained": d["bf16_tflops_sustained"],
                "source": "measured"}
    # NVIDIA's H100 SXM data sheet (700 W card, dense BF16): an upper bound, not a measured rate
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "source": "H100 SXM data sheet"}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region (read-only queries)."""

    def __init__(self, index: int):
        self.index, self.rows, self._stop = index, [], threading.Event()
        self.t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.rows.append([c.strip() for c in out.split(",")])
            except Exception:
                pass
            self._stop.wait(0.2)

    def __enter__(self):
        self.t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self.t.join(timeout=3)

    def summary(self):
        sm, mx, reasons = [], 0.0, set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[0]))
                mx = max(mx, float(r[1]))
                for n, v in zip(names, r[3:7]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
            except Exception:
                continue
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx or None, "reasons": sorted(reasons),
                "samples": len(sm)}


# ====================================================================== CPU arm (oracle port)
def best_cpu_threads() -> int:
    """torch CPU eager oversubscribes badly on many-core hosts (128 threads ran 250x slower than 8 on
    this path); pick the fastest of a few thread counts on one frame, as a fair reference arm would."""
    n = os.cpu_count() or 1
    best, best_v = 1, 0.0
    for t in sorted({min(n, c) for c in (8, 16, 32)}):
        v, _ = cpu_sample(4, 1, t)
        if v > best_v:
            best, best_v = t, v
    return best


def cpu_sample(streams: int, frames: int, threads: int):
    """The reference's CPU path (oracle restatement, torch CPU fp32): streaming encode+decode."""
    import torch
    from oracle import mimi_oracle as O
    from specs import mimi_spec as S
    torch.set_num_threads(threads)
    w = S.synthetic_weights(S.OFFICIAL, seed=41)
    x = S.synthetic_audio(streams, FRAME * (frames + 1), seed=0)
    sc = O.StreamingCodec(w, streams)
    with torch.no_grad():
        c = sc.encode(x[..., :FRAME])  # warm-up frame
        sc.decode(c)
        t0 = time.perf_counter()
        for i in range(1, frames + 1):
            c = sc.encode(x[..., i * FRAME:(i + 1) * FRAME])
            sc.decode(c)
        dt = time.perf_counter() - t0
    return streams * frames / dt, dt


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    threads = best_cpu_threads()
    streams, frames = 64, 2     # 64 streams: a quarter of the product arm's batch (torch CPU at 8 streams is overhead-bound)
    cpu_sample(streams, 1, threads)
    for _ in range(max(0, args.warmup - 1)):
        cpu_sample(streams, 1, threads)
    t0 = time.perf_counter()
    vals = []
    for _ in range(args.steps):
        v, _ = cpu_sample(streams, frames, threads)
        vals.append(v)
    dt = time.perf_counter() - t0
    value = sum(vals) / len(vals)
    sample = f"{streams} streams x {frames} frames per step (streaming, 1 warm-up frame), torch CPU fp32"
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": WORKLOAD, "streams_per_gpu": STREAMS, "frames_per_stream": FRAMES},
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": threads, "host_cores": os.cpu_count(), "kind": "port",
                         "sample": sample},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


# ====================================================================== GPU arm
def run_ours(args):
    import torch
    import torch.distributed as dist
    from specs import mimi_spec as S   # seeded synthetic weights / audio (neutral spec module; nothing from oracle/ here)
    from rstnet_b200 import _lib, ops
    from rstnet_b200.codec import MimiCodec
    from rstnet_b200.dist import reduce_timing

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "bench.py needs a GPU (no CPU fallback; use --impl reference for the CPU arm)"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        if os.environ.get("NCCL_DEBUG", "").upper() in ("", "VERSION"):
            os.environ["NCCL_DEBUG"] = "WARN"      # NCCL's version banner goes to stdout: keep the one-JSON-line contract
        dist.init_process_group("nccl", device_id=dev)

    m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
    m = m.to(dev).eval()
    m.use_cuda_graphs = True
    B = STREAMS
    # 10 s of audio per stream: 4 distinct seeded clips tiled over the batch, plus per-rank offset
    base = S.synthetic_audio(8, FRAME * FRAMES, seed=100 + rank)
    host = base.repeat(B // 8, 1, 1).contiguous()                      # [B,1,240000]
    x_dev = host.to(dev)                                               # resident copy for `value`
    # e2e arm: audio arrives as 80 ms chunks (one per stream per step), each chunk contiguous in pinned host memory
    host_frames = host.view(B, 1, FRAMES, FRAME).permute(2, 0, 1, 3).contiguous().pin_memory()   # [FRAMES,B,1,1920]
    out_wav_host = torch.empty(B, 1, FRAME, dtype=torch.float32).pin_memory()
    out_codes_host = torch.empty(B, 8, 1, dtype=torch.int64).pin_memory()

    state = {"entered": False}
    # --dump-outputs: what every frame of a step returned (tokens of every stream, the waveform of a fixed seeded sample
    # of streams), collected by an untimed replay of the last timed step (see run_ours), never inside the timed region
    dump = {"on": False, "codes": [], "wav": []}
    wav_rows = torch.randperm(B, generator=torch.Generator().manual_seed(0))[:32].sort().values
    wav_rows_dev = wav_rows.to(dev)

    def step(resident: bool, cold: bool = True):
        """125 streaming frames for all streams: encode chunk -> decode tokens.  One streaming scope is
        kept for the whole run (buffers + CUDA graphs are reused) and reset between passes (cold = every pass starts
        like a new 10 s stream; cold False keeps the state: the transformer rings stay full)."""
        if state["entered"] and cold:
            m.reset_streaming()
        state["entered"] = True
        for i in range(FRAMES):
            if resident:
                chunk = x_dev[..., i * FRAME:(i + 1) * FRAME]
            else:
                chunk = host_frames[i].to(dev, non_blocking=True)
            codes = m.encode(chunk)
            wav = m.decode(codes)
            state["last"] = (codes, wav)
            if dump["on"]:
                dump["codes"].append(codes.clone())
                dump["wav"].append(wav.index_select(0, wav_rows_dev))
            if not resident:
                out_codes_host.copy_(codes, non_blocking=True)
                out_wav_host.copy_(wav, non_blocking=True)
        if not resident:
            torch.cuda.current_stream().synchronize()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(resident: bool, steps: int, cold: bool = True):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        l0 = _lib.launch_count()
        e0.record()
        for _ in range(steps):
            step(resident, cold)
        e1.record()
        barrier()
        ms, _ = reduce_timing(e0.elapsed_time(e1), B * FRAMES * steps, device=dev)  # max over ranks
        return ms, _lib.launch_count() - l0

    # launches per frame (eager count; graph replays re-issue exactly these nodes)
    m.use_cuda_graphs = False
    m.streaming_forever(B)
    l0 = _lib.launch_count()
    c = m.encode(x_dev[..., :FRAME])
    m.decode(c)
    launches_per_frame = _lib.launch_count() - l0
    m.use_cuda_graphs = True
    m.streaming_forever(B)
    state["entered"] = False

    for _ in range(max(3, args.warmup)):
        step(True)
    with ClockSampler(local) as cs:
        ms, _ = timed(True, args.steps)
    clocks = cs.summary()
    if args.dump_outputs and rank == 0:
        # Every timed step is a cold pass over the same inputs, so an untimed replay of one computes what the last timed
        # step computed; the replay's last frame is checked bit for bit against the last frame the timed run returned.
        import numpy as np
        last_codes, last_wav = (t.clone() for t in state["last"])
        dump["on"] = True
        step(True)
        dump["on"] = False
        assert torch.equal(dump["codes"][-1], last_codes) and torch.equal(dump["wav"][-1], last_wav.index_select(0, wav_rows_dev)), \
            "the untimed replay differs from the last timed step"
        os.makedirs(args.dump_outputs, exist_ok=True)
        codes_all = torch.stack(dump["codes"]).reshape(FRAMES, B, 8).permute(1, 2, 0)             # [B, 8, FRAMES]
        wav_all = torch.stack(dump["wav"]).reshape(FRAMES, len(wav_rows), FRAME).permute(1, 0, 2)  # [32, FRAMES, 1920]
        np.save(os.path.join(args.dump_outputs, "codes.npy"), codes_all.float().cpu().numpy())
        np.save(os.path.join(args.dump_outputs, "wav.npy"), wav_all.reshape(len(wav_rows), -1).float().cpu().numpy())
        np.save(os.path.join(args.dump_outputs, "wav_streams.npy"), wav_rows.float().numpy())
        dump["codes"].clear()
        dump["wav"].clear()
    for _ in range(1):
        step(False)
    ms_e2e, _ = timed(False, args.steps)
    # steady state: no reset between passes -> after the pass above the 250-token rings are full for every frame
    step(True, cold=False)
    ss_steps = max(1, min(args.steps, 4))
    ms_ss, _ = timed(True, ss_steps, cold=False)

    frames_total = world * B * FRAMES * args.steps
    value = frames_total / (ms / 1e3)
    e2e_value = frames_total / (ms_e2e / 1e3)
    ss_value = world * B * FRAMES * ss_steps / (ms_ss / 1e3)

    if rank == 0:
        roof = roofline_pass(m, x_dev, B, dev)
        cpu = None
        extras = {}
        if world == 1:   # reported baseline: rank 0 at N = 1 only
            cpu_threads = best_cpu_threads()
            cv8, cdt8 = cpu_sample(8, 4, cpu_threads)
            cv, cdt = cpu_sample(64, 2, cpu_threads)
            cpu = {"value": cv, "unit": UNIT, "cores": cpu_threads, "host_cores": os.cpu_count(), "kind": "port",
                   "sample": f"64 streams x 2 frames streaming encode+decode, torch CPU fp32 oracle port ({cdt:.1f} s); "
                             f"8 streams x 4 frames gives {cv8:.0f} frames/s"}
        lm = None
        if world == 1 and not args.no_lm:
            def guarded(name, fn):
                try:   # the codec headline must not be lost to a failure in a secondary measurement
                    extras[name] = fn()
                except Exception as e:
                    extras[name] = {"error": f"{type(e).__name__}: {e}"[:300]}
                gc.collect()              # streaming states hold reference cycles (plans <-> closures): free their HBM now
                torch.cuda.empty_cache()
            guarded("gpu_eager_codec", lambda: gpu_eager_codec_baseline(dev, B))
            m._stream_state = None
            m._engine = None
            torch.cuda.empty_cache()
            guarded("lm_decode", lambda: lm_decode_bench(dev, steps=10, warmup=3))
            lm = extras.pop("lm_decode")
            guarded("cfg4_infer", lambda: cfg4_infer_bench(dev, S))
            guarded("cfg5_duplex", lambda: cfg5_duplex_bench(dev, S))
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps, "warmup": max(3, args.warmup),
            "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": WORKLOAD, "streams_per_gpu": B, "frames_per_stream": FRAMES, "frame_samples": FRAME,
                       "codec_only_realtime_streams_per_gpu": value / world / 12.5, "cuda_graphs": True,
                       "start": "cold (every pass = new 10 s streams: the transformer rings fill from empty)",
                       "l2_policy": "inputs larger than L2 (246 MB audio + 320 MB weights per pass)",
                       "parallelism": f"dp{world}"},
            "clocks": clocks,
            "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": B * FRAME * FRAMES * 4,
                    "d2h_bytes_per_step": B * FRAMES * (FRAME * 4 + 8 * 8), "ms_per_step": ms_e2e / args.steps},
            "gpu_launches": int(launches_per_frame * FRAMES * args.steps),
            "roofline": roof,
            "steady_state": {"value": ss_value, "unit": UNIT, "ms_per_step": ms_ss / ss_steps, "steps": ss_steps,
                             "codec_only_realtime_streams_per_gpu": ss_value / world / 12.5,
                             "note": "same pass without reset: every frame attends a full 250-token ring (long-running server)"},
            "lm_decode": lm,
            "cpu_baseline": cpu,
        }
        if extras:
            eager = extras.pop("gpu_eager_codec", None)
            lm_eager = (lm or {}).pop("gpu_eager", None) if isinstance(lm, dict) else None
            line["gpu_eager_baseline"] = {"codec": eager, "lm_decode": lm_eager,
                                          "what": "the reference's eager arithmetic (oracle port = the same ATen calls) on this GPU"}
            if isinstance(eager, dict) and eager.get("value"):
                line["gpu_eager_baseline"]["codec_speedup"] = value / eager["value"]
            line.update(extras)
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def roofline_pass(m, x_dev, B, dev):
    """Dominant kernel = gemm_tc_kernel (persistent wgmma 3xTF32 GEMM; every conv / transposed conv /
    linear of a frame).  Per-launch CUDA-event timing of each launch over a few eager streaming frames
    (events on the launching stream).  Each frame is queued behind a ~10 ms spin kernel so the host stays
    ahead of the device and the event pairs bracket device time, not host launch latency.
    achieved = algorithmic FLOPs (2*M*N*K per launch, one fp32-equivalent product per MAC -- the 3 TF32
    MMAs that implement it are not counted) / summed launch time."""
    import torch
    from rstnet_b200 import ops
    peaks = _peaks()
    rec, rec_bytes = [], []
    orig = ops.TcGemm.run

    def timed_run(self):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        orig(self)
        e1.record()
        rec.append((e0, e1, self.flops))
        rec_bytes.append(self.bytes)

    m.use_cuda_graphs = False
    ops.TcGemm.run = timed_run  # plans bind `run` when they are built, so patch before the scope is created
    try:
        m.streaming_forever(B)
        c = m.encode(x_dev[..., :FRAME])
        m.decode(c)  # untimed warm frame
        torch.cuda.synchronize()
        rec.clear()
        rec_bytes.clear()
        nframes = 3
        frame_ev = []
        for j in range(1, 1 + nframes):
            i = j % FRAMES
            torch.cuda._sleep(20_000_000)   # ~10 ms: the whole frame is enqueued before the device starts it
            f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            f0.record()
            c = m.encode(x_dev[..., i * FRAME:(i + 1) * FRAME])
            m.decode(c)
            f1.record()
            frame_ev.append((f0, f1))
        torch.cuda.synchronize()
        frame_ms = sum(a.elapsed_time(b) for a, b in frame_ev)
    finally:
        ops.TcGemm.run = orig
        m.use_cuda_graphs = True
    t_ms = sum(a.elapsed_time(b) for a, b, _ in rec)
    flops = sum(f for _, _, f in rec)
    achieved = flops / (t_ms * 1e-3) / 1e12
    peak = peaks["bf16_tflops_sustained"]
    alg_bytes = sum(b for b in rec_bytes) / max(1, len(rec_bytes))     # per launch, like `traffic`
    return {"bound": "tensor", "kernel": "gemm_tc_kernel (persistent wgmma tf32 GEMM, A fragments in registers, 3xTF32 split = fp32-equivalent; all conv/linear launches of a frame)",
            "achieved": achieved, "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak,
            "algorithmic_bytes_per_launch": alg_bytes,
            "frac_of_3xtf32_ceiling": achieved / (peak / 6.0),
            "peak_source": f"{peaks['source']} dense bf16 (TF32 dense peak is half of it; 3xTF32 issues 3 MMAs per product, so the ceiling of this metric is peak/6)",
            "launches": len(rec) // nframes, "avg_launch_us": 1e3 * t_ms / max(1, len(rec)),
            "share_of_frame_time": t_ms / frame_ms, "eager_frame_ms": frame_ms / nframes,
            "gflop_per_frame_batch": flops / nframes / 1e9}


def lm_decode_bench(dev, steps: int, warmup: int):
    """BASELINE.json configs[2]: one decode step (temporal 32-layer 7B + 8 depth steps + sampling) of the
    speech-text LM, random-init bf16 weights, batch 32 streams, KV ring pre-filled to 2048 positions (a stream's 7B MHA ring
    costs 1.07 GB: 64 of them would not fit next to the 17 GB of weights in 80 GB).
    Reported next to the codec headline (it is a different unit of work, not part of `value`)."""
    import torch
    from rstnet_b200 import _lib, ops
    from rstnet_b200 import lm as LMmod
    from rstnet_b200.lm import GPT, Config
    peaks = _peaks()
    B, KV = 32, 2048
    cfg = Config(block_size=4096, n_layer=32, n_embd=4096, n_head=32, head_size=128, intermediate_size=11008,
                 padded_vocab_size=152064, audio_card=2050, n_q=8, dep_q=8, codecformer_dim=1024, codecformer_heads=16,
                 codecformer_layers=6, codecformer_dim_feedforward=4224, context=KV)
    m = GPT(cfg, device=dev, dtype=torch.bfloat16).eval()
    n_params = sum(p.numel() for p in m.parameters())
    # per-launch accounting hooks (bound when the scope's plans are built)
    rec = {"gemm": [], "attn": []}
    timing = {"on": False}
    orig_run = LMmod.SkinnyGemm.run
    L = _lib.lib()
    orig_attn = L.rstnet_lm_ring_decode_attention_bf16

    def timed_run(self):
        if not timing["on"]:
            return orig_run(self)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); orig_run(self); e1.record()
        rec["gemm"].append((e0, e1, self.bytes, tuple(self._keep[1].shape)))

    def timed_attn(*a):
        if not timing["on"]:
            return orig_attn(*a)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); r = orig_attn(*a); e1.record()
        rec["attn"].append((e0, e1, 2.0 * B * cfg.n_head * (KV - 1) * cfg.head_size * 2))
        return r

    LMmod.SkinnyGemm.run = timed_run
    L.rstnet_lm_ring_decode_attention_bf16 = timed_attn
    try:
        m.streaming_forever(B)
        st = m._state
        for kv in st.kv:
            kv.normal_()
        st.offset.fill_(KV + 8)  # ring already wrapped: every step attends the full window
        st.pos_host[:] = KV + 8
        g = torch.Generator(device=dev).manual_seed(0)
        seq = torch.randint(0, 2048, (B, 9, 1), device=dev, generator=g)
        seq[:, 0] = torch.randint(0, 128256, (B, 1), device=dev, generator=g)
        host_seq = seq.cpu().pin_memory()
        host_tok = torch.empty(B, 9, dtype=torch.int64).pin_memory()
        m.use_cuda_graphs = True
        for _ in range(max(3, warmup)):
            m.forward_step(seq)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            m.forward_step(seq)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        e0.record()
        for _ in range(steps):
            t = m.forward_step(host_seq.to(dev, non_blocking=True))
            host_tok.copy_(t, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        e1.record()
        torch.cuda.synchronize()
        ms_e2e = e0.elapsed_time(e1) / steps
        # in-graph split of the step: the temporal transformer's own graph, replayed alone (position rewound each time
        # so it keeps attending the full window); the rest of the frame graph is the depth transformer + sampling
        n_t = max(3, steps)
        for i in range(n_t + 2):
            if i == 2:
                torch.cuda.synchronize()
                e0.record()
            st._replay(("temporal",), st._temporal)
            st.offset.fill_(KV + 8)
        e1.record()
        torch.cuda.synchronize()
        ms_temporal = e0.elapsed_time(e1) / n_t
        st.pos_host[:] = KV + 8
        # per-kernel roofline pass: one eager frame with events around every GEMM / attention launch
        m.use_cuda_graphs = False
        m.forward_step(seq)
        timing["on"] = True
        m.forward_step(seq)
        torch.cuda.synchronize()
        timing["on"] = False
    finally:
        LMmod.SkinnyGemm.run = orig_run
        L.rstnet_lm_ring_decode_attention_bf16 = orig_attn

    def agg(items):
        t = sum(it[0].elapsed_time(it[1]) for it in items)
        by = sum(it[2] for it in items)
        return {"launches": len(items), "ms": t, "gbytes": by / 1e9, "achieved_gbs": by / 1e9 / (t * 1e-3) if t else None,
                "frac": (by / 1e9 / (t * 1e-3)) / peaks["hbm_gbs"] if t else None}

    w_bytes = 2.0 * n_params - 2.0 * (152064 * 4096 + 8 * 2051 * 4096 + 152064 * 1024 + 7 * 2051 * 1024)  # embeddings are gathered, not streamed
    kv_bytes = 32 * 2.0 * B * 32 * (KV - 1) * 128 * 2
    step_bytes = w_bytes + kv_bytes
    out = {"workload": f"gpt7b_decode_step_B{B}_kv{KV} (32-layer temporal + 8x6-layer depth + sampling)", "dtype": "bf16",
           "params": n_params, "ms_per_step": ms, "frames_per_s": B / (ms * 1e-3), "tokens_per_s": B * 9 / (ms * 1e-3),
           "e2e_ms_per_step": ms_e2e, "e2e_tokens_per_s": B * 9 / (ms_e2e * 1e-3),
           "algorithmic_gbytes_per_step": step_bytes / 1e9,
           "roofline": {"bound": "hbm", "achieved": step_bytes / 1e9 / (ms * 1e-3), "peak": peaks["hbm_gbs"], "unit": "GB/s",
                        "frac": step_bytes / 1e9 / (ms * 1e-3) / peaks["hbm_gbs"], "peak_source": peaks["source"]},
           "attention_kernel": agg(rec["attn"]), "gemm_kernels": agg(rec["gemm"])}
    att_ms = out["attention_kernel"]["ms"]
    tw = 2.0 * (cfg.n_layer * (3 * cfg.n_embd * cfg.n_embd + cfg.n_embd * cfg.n_embd + 3 * cfg.n_embd * cfg.intermediate_size)
                + cfg.padded_vocab_size * cfg.n_embd)      # qkv + proj + (fc_1, fc_2, down) per layer + the text head, bf16
    rest = ms_temporal - att_ms
    out["in_graph_split_ms"] = {
        "temporal_graph": ms_temporal, "attention_32_layers": att_ms, "temporal_gemms_and_small_kernels": rest,
        "depth_transformer_and_sampling": ms - ms_temporal, "temporal_weight_gbytes": tw / 1e9,
        "temporal_gemm_in_graph_gbs": tw / 1e9 / (rest * 1e-3) if rest > 0 else None,
        "temporal_gemm_in_graph_frac": tw / 1e9 / (rest * 1e-3) / peaks["hbm_gbs"] if rest > 0 else None,
        "note": "temporal_graph = the temporal transformer's CUDA graph replayed alone; the eager per-launch GEMM times above include "
                "event / launch overhead and understate the in-graph rate; the in-graph figure charges the GEMMs with every "
                "finalize / RoPE / embedding launch of the temporal part"}
    shapes = {}
    for it in rec["gemm"]:
        d = shapes.setdefault(str(it[3]), [0, 0.0, 0.0])
        d[0] += 1; d[1] += it[0].elapsed_time(it[1]); d[2] += it[2]
    out["gemm_by_shape_NK"] = {k: {"launches": v[0], "avg_us": 1e3 * v[1] / v[0], "gbs": v[2] / 1e9 / (v[1] * 1e-3)} for k, v in shapes.items()}
    m._state = None
    m._packed = None
    torch.cuda.empty_cache()
    # same-box comparator (BASELINE.md §4): the reference's eager arithmetic on this GPU -- the oracle port executes the
    # ATen calls of models/llama_streaming.py (F.linear, index_copy_ ring, boolean-mask SDPA over the whole ring, ...) in
    # bf16 on the same weights, one launch per op, no CUDA graph (utils/compile.py's CUDAGraphed wraps only Moshi's LMGen)
    try:
        from oracle import lm_oracle as LO
        ocfg = LO.LMConfig(context=KV, block_size=4096)
        w = {k: v.detach() for k, v in m.state_dict().items()}
        gs = LO.GPTStream(w, ocfg, B)
        for r in gs.rings:
            r.cache.normal_()
            r.end_offset = KV + 8
        gs.offset = KV + 8
        with torch.no_grad():
            LO.greedy_frame(gs, seq)
            torch.cuda.synchronize()
            e0.record()
            n_e = 3
            for _ in range(n_e):
                LO.greedy_frame(gs, seq)
            e1.record()
            torch.cuda.synchronize()
        ems = e0.elapsed_time(e1) / n_e
        out["gpu_eager"] = {"ms_per_step": ems, "tokens_per_s": B * 9 / (ems * 1e-3), "speedup": ems / ms,
                            "what": "oracle port (reference ATen calls) in bf16 on this GPU, greedy frame, eager"}
        del gs, w
    except Exception as e:
        out["gpu_eager"] = {"error": f"{type(e).__name__}: {e}"[:300]}
    del m
    torch.cuda.empty_cache()
    return out


def gpu_eager_codec_baseline(dev, B):
    """The reference's eager codec arithmetic on this GPU: the oracle's StreamingCodec (F.conv1d / conv_transpose1d /
    F.linear / SDPA / cdist+argmin, one ATen call per op as MLLM_v2/modules does; PyTorch's default conv TF32 setting) with
    the weights on the device, streaming, same batch as the headline.  Bounded sample: 1 warm-up + 5 timed frames."""
    import torch
    from oracle import mimi_oracle as O
    from specs import mimi_spec as S
    w = {k: v.to(dev) for k, v in S.synthetic_weights(S.OFFICIAL, seed=41).items()}
    x = S.synthetic_audio(8, FRAME * 6, seed=3).repeat(B // 8, 1, 1).to(dev)
    sc = O.StreamingCodec(w, B)
    with torch.no_grad():
        c = sc.encode(x[..., :FRAME]); sc.decode(c)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(1, 6):
            c = sc.encode(x[..., i * FRAME:(i + 1) * FRAME]); sc.decode(c)
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    return {"value": B * 5 / (ms * 1e-3), "unit": UNIT, "ms_per_frame_batch": ms / 5,
            "sample": f"{B} streams x 5 frames (cold start), torch eager fp32 (conv TF32 default: "
                      f"{torch.backends.cudnn.allow_tf32})"}


def _gpt7b(dev, context):
    import torch
    from rstnet_b200.lm import GPT, Config
    cfg = Config(block_size=4096, n_layer=32, n_embd=4096, n_head=32, head_size=128, intermediate_size=11008,
                 padded_vocab_size=152064, audio_card=2050, n_q=8, dep_q=8, codecformer_dim=1024, codecformer_heads=16,
                 codecformer_layers=6, codecformer_dim_feedforward=4224, context=context)
    return GPT(cfg, device=dev, dtype=torch.bfloat16).eval()


def _mimi(dev, S):
    from rstnet_b200.codec import MimiCodec
    m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
    return m.to(dev).eval()


def cfg4_infer_bench(dev, S, B: int = 32, prompt_frames: int = 50, gen_frames: int = 1000):
    """BASELINE configs[3] (infer_no_streaming.py end to end): Mimi encode of the prompt audio -> InferenceImp (prefill of the
    prompt, then `gen_frames` generated frames: temporal step + 8 depth steps + sampling each) -> reverse_delay -> Mimi
    decode of everything generated; 7B random-init LM in bf16, B = 32 utterances, temp 0.8 / 0.7, top-k 30 / 25.
    The prompt audio and the decoded waveforms cross PCIe inside the timed region."""
    import torch
    from rstnet_b200.infer import InferenceImp
    codec = _mimi(dev, S)
    lm = _gpt7b(dev, context=2048)
    imp = InferenceImp(None, lm, "sampling", 0.7, 25, 0.8, 30, "TTS")
    audio_host = S.synthetic_audio(8, FRAME * prompt_frames, seed=9).repeat(B // 8, 1, 1).pin_memory()
    g = torch.Generator().manual_seed(4)
    text = torch.randint(0, 128000, (B, prompt_frames), generator=g)

    def run(n_gen):
        t = {}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        codes = codec.encode(audio_host.to(dev, non_blocking=True))                     # [B, 8, P]
        seq = torch.full((B, 9, prompt_frames + n_gen), 128002, dtype=torch.int64, device=dev)   # text-empty = to generate
        seq[:, 0, :prompt_frames] = text.to(dev)
        seq[:, 1:, :prompt_frames] = codes
        seq[:, 1:, prompt_frames:] = 0
        ev[1].record()
        out = imp.generate(seq)                                                         # [B, 8, n_gen - 1]
        ev[2].record()
        wav = codec.decode(out.clamp(max=2047))
        wav_host = wav.cpu()
        ev[3].record()
        torch.cuda.synchronize()
        return [ev[i].elapsed_time(ev[i + 1]) for i in range(3)], out, wav_host

    run(8)                                   # warm-up: builds plans, captures the frame graphs
    (t_enc, t_gen, t_dec), out, wav = run(gen_frames)
    total = (t_enc + t_gen + t_dec) * 1e-3
    res = {"workload": f"mimi_encode_{prompt_frames}f -> InferenceImp prefill+{gen_frames} frames -> mimi_decode, B={B}, 7B bf16 random init",
           "seconds": {"encode_prompt": t_enc * 1e-3, "generate": t_gen * 1e-3, "decode": t_dec * 1e-3, "total": total},
           "tokens_per_s": B * 9 * gen_frames / total, "frames_per_s": B * gen_frames / total,
           "generate_ms_per_frame": t_gen / gen_frames, "audio_seconds_generated": B * (gen_frames - 1) * 0.08,
           "realtime_factor": B * (gen_frames - 1) * 0.08 / total,
           "h2d_bytes": int(audio_host.numel() * 4), "d2h_bytes": int(wav.numel() * 4), "codes_shape": list(out.shape)}
    lm._state = None
    del lm, codec, imp
    return res


def cfg5_duplex_bench(dev, S, ticks: int = 40):
    """BASELINE configs[4] on ONE GPU: B concurrent dialogue streams through rstnet_b200.serve.DuplexEngine -- per 80 ms
    tick: H2D of every stream's 1920-sample chunk, codec encode, one 7B LM frame (temporal + depth + sampling), codec
    decode, D2H of tokens + PCM (the loop of moshi/server.py:108-144 for a batch).  Reports the wall-clock latency of a
    tick (p50 / p99 over `ticks` ticks after warm-up) and which batch sizes stay under the 80 ms real-time budget.  The
    7B MHA KV ring (context 2048, bf16) costs 1.07 GB per stream, which is what bounds streams per GPU (SURVEY.md H4):
    with the 17 GB of weights roughly 55 streams' rings fit in 80 GB; the batches tried stay below that, so the reported
    streams per GPU is a lower bound."""
    import torch
    from rstnet_b200.serve import DuplexEngine, FrameScheduler
    codec = _mimi(dev, S)
    lm = _gpt7b(dev, context=2048)
    res = {"tick_budget_ms": 80.0, "runs": []}
    audio = S.synthetic_audio(8, FRAME * 8, seed=12)
    for B in (32, 48):
        try:
            eng = DuplexEngine(codec, lm, B)
            sch = FrameScheduler(eng, B)
            for s in range(B):
                sch.admit(s)
            for tick in range(ticks + 6):
                if tick == 3:
                    # long-running sessions: every ring full from here on (LM: 2048-key window per stream, random K/V so the
                    # softmax is not degenerate; codec: 250-token windows) -- a fresh session's first seconds are cheaper
                    st = lm._state
                    for kv in st.kv:
                        kv.normal_()
                    st.offset.fill_(2048 + 100); st.pos_host[:] = 2048 + 100
                    for plan in list(codec._stream_state.enc.values()) + list(codec._stream_state.dec.values()):
                        plan.offset.fill_(1000)
                for s in range(B):
                    sch.push(s, audio[s % 8, 0, (tick % 8) * FRAME:(tick % 8 + 1) * FRAME])
                out = sch.tick()
                assert len(out) == B
            lat = sorted(eng.latencies_ms[6:])
            p = lambda q: lat[min(len(lat) - 1, int(q * len(lat)))]
            res["runs"].append({"streams": B, "tick_ms_p50": p(0.5), "tick_ms_p99": p(0.99), "tick_ms_max": lat[-1],
                                "realtime": p(0.99) < 80.0, "frames_per_s": B / (p(0.5) * 1e-3),
                                "headroom_x": 80.0 / p(0.5)})
        except torch.cuda.OutOfMemoryError as e:
            res["runs"].append({"streams": B, "error": "out of memory (KV rings)"})
        lm._state = None
        codec._stream_state = None
        eng = sch = st = plan = kv = out = None      # every local that still points into the scope's HBM
        gc.collect()
        torch.cuda.empty_cache()
    ok = [r["streams"] for r in res["runs"] if r.get("realtime")]
    res["realtime_streams_per_gpu"] = max(ok) if ok else 0
    res["state"] = "steady: LM KV rings full (2048-key window, wrapped), codec transformer rings full (250 tokens)"
    res["note"] = ("codec + 7B LM per stream at an 80 ms cadence; the largest batch tried that keeps p99 < 80 ms (a lower bound) "
                   "(48 streams = ~51 GB of MHA KV rings next to the weights)")
    del lm, codec
    return res


def main():
    global FRAMES, WORKLOAD
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-lm", dest="no_lm", action="store_true", help="skip the secondary LM decode-step measurement")
    ap.add_argument("--dump-outputs", dest="dump_outputs", default=None, metavar="DIR",
                    help="write the outputs of the last timed step as DIR/<name>.npy (float32)")
    ap.add_argument("--frames", type=int, default=FRAMES,
                    help="frames per stream per step (profiling aid: a short pass; the default 125 is the bench)")
    args = ap.parse_args()
    if args.frames != FRAMES:
        FRAMES = args.frames
        WORKLOAD += f"_SHORT{FRAMES}frames"
    if args.impl == "reference":
        run_reference(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()
