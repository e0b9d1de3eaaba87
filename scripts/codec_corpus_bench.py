"""Corpus tokenization throughput of the codec: MimiCodec.encode_many / decode_many (continuous batching of ragged clips)
against today's per-clip drivers, on a seeded synthetic corpus (clip lengths uniform in 1 s .. 40 s, 24 kHz) and the
seeded weights of specs/.  Prints one JSON line:

  * encode_many at each capacity x chunk length (12.5 Hz frames per step): audio-seconds/s, frames/s and row occupancy
    (clip chunks computed / (steps x capacity), from the admission schedule);
  * decode_many at each capacity x chunk length;
  * offline.tokenize_utterances and per-clip decode on the first --baseline-clips clips (each clip has its own length, so
    each is its own batch), and the code frames / max waveform difference between the two paths on those clips;
  * the card's name and power limit, read in the same call.

Times are host wall clock from a device synchronise to the end of the call, plan set-up and graph capture included.

usage: python scripts/codec_corpus_bench.py [--clips 1024] [--baseline-clips N] [--capacities 64,128,256]
                                            [--chunks 1,2,4,8] [--seed 0] [--out FILE]
"""
import argparse
import heapq
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rstnet_b200 import codec as codec_mod      # noqa: E402
from rstnet_b200 import offline                 # noqa: E402
from specs import mimi_spec as S                # noqa: E402

SR, FS = 24000, 1920


def corpus(n, seed):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1 * SR, 40 * SR + 1, size=n)
    return [(f"utt{i:04d}", S.synthetic_audio(1, int(L), seed=seed * 100003 + i)[0, 0]) for i, L in enumerate(lengths)]


def occupancy(steps_per_clip, capacity):
    """(steps, occupancy) of the admission schedule: row b takes the next clip the step after its clip's last one."""
    rows = [(0, b) for b in range(capacity)]       # (first free step, row)
    heapq.heapify(rows)
    end = 0
    for n in steps_per_clip:
        t, b = heapq.heappop(rows)
        heapq.heappush(rows, (t + n, b))
        end = max(end, t + n)
    return end, sum(steps_per_clip) / (end * capacity)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the name from the driver is still worth reporting
        q = f"nvidia-smi unavailable ({e})"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1024)
    ap.add_argument("--baseline-clips", type=int, default=None, help="default: every clip")
    ap.add_argument("--capacities", default="64,128,256")
    ap.add_argument("--chunks", default="1,2,4,8")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = "cuda"
    caps = [int(c) for c in args.capacities.split(",")]
    chunks = [int(c) for c in args.chunks.split(",")]
    m = codec_mod.MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
    m = m.to(dev).eval()
    clips = corpus(args.clips, args.seed)
    lengths = [w.numel() for _, w in clips]
    audio_s = sum(lengths) / SR
    frames = sum(math.ceil(L / FS) for L in lengths)
    res = {"card": card(), "clips": args.clips, "audio_seconds": round(audio_s, 1), "frames": frames, "encode_many": [],
           "decode_many": []}
    default_chunk = codec_mod.CORPUS_CHUNK_FRAMES

    # warm-up: module load, kernel attributes, allocator
    list(m.encode_many(clips[:4], 4))

    codes_by_cfg = {}
    for ch in chunks:
        codec_mod.CORPUS_CHUNK_FRAMES = ch
        for cap in caps:
            codes, dt = timed(lambda: dict(m.encode_many(clips, cap)))
            steps, occ = occupancy([math.ceil(L / (ch * FS)) for L in lengths], cap)
            res["encode_many"].append({"capacity": cap, "chunk_frames": ch, "seconds": round(dt, 3),
                                       "audio_s_per_s": round(audio_s / dt, 1), "frames_per_s": round(frames / dt, 1),
                                       "steps": steps, "occupancy": round(occ, 4)})
            print(json.dumps(res["encode_many"][-1]), file=sys.stderr)
            codes_by_cfg[(cap, ch)] = codes
    ref_cfg = (max(caps), default_chunk) if (max(caps), default_chunk) in codes_by_cfg else next(iter(codes_by_cfg))
    ref = codes_by_cfg[ref_cfg]
    res["code_frames_differing_between_encode_many_configs"] = {
        f"cap{cap}_chunk{ch}": int(sum(int((c[k] != ref[k]).any(dim=0).sum()) for k in ref))
        for (cap, ch), c in codes_by_cfg.items()}

    code_items = [(k, ref[k]) for k, _ in clips]
    wavs = None
    for ch in chunks:
        codec_mod.CORPUS_CHUNK_FRAMES = ch
        for cap in caps:
            out, dt = timed(lambda: dict(m.decode_many(code_items, cap)))
            steps, occ = occupancy([math.ceil(c.shape[1] / ch) for _, c in code_items], cap)
            res["decode_many"].append({"capacity": cap, "chunk_frames": ch, "seconds": round(dt, 3),
                                       "audio_s_per_s": round(audio_s / dt, 1), "frames_per_s": round(frames / dt, 1),
                                       "steps": steps, "occupancy": round(occ, 4)})
            print(json.dumps(res["decode_many"][-1]), file=sys.stderr)
            if (cap, ch) == ref_cfg:
                wavs = out
            del out
    codec_mod.CORPUS_CHUNK_FRAMES = default_chunk

    # today's per-clip drivers on the first clips: every clip its own length, so its own batch (B = 1, CUDA cores)
    nb = args.clips if args.baseline_clips is None else min(args.baseline_clips, args.clips)
    base = clips[:nb]
    b_audio = sum(w.numel() for _, w in base) / SR
    b_frames = sum(math.ceil(w.numel() / FS) for _, w in base)
    offline.tokenize_utterances(m, base[:2])   # warm-up
    toks, dt = timed(lambda: offline.tokenize_utterances(m, base))
    res["tokenize_utterances"] = {"clips": nb, "seconds": round(dt, 3), "audio_s_per_s": round(b_audio / dt, 1),
                                  "frames_per_s": round(b_frames / dt, 1)}
    res["code_frames_differing_from_tokenize_utterances"] = {
        "config": f"cap{ref_cfg[0]}_chunk{ref_cfg[1]}", "frames": b_frames,
        "differing": int(sum(int((toks[k].long() != ref[k]).any(dim=0).sum()) for k, _ in base))}

    def per_clip_decode(part):
        return {k: m.decode(ref[k][None].to(dev))[0, 0].cpu() for k, _ in part}
    per_clip_decode(base[:2])   # warm-up
    dwav, dt = timed(lambda: per_clip_decode(base))
    res["per_clip_decode"] = {"clips": nb, "seconds": round(dt, 3), "audio_s_per_s": round(b_audio / dt, 1),
                              "frames_per_s": round(b_frames / dt, 1)}
    res["decode_many_config"] = f"cap{ref_cfg[0]}_chunk{ref_cfg[1]}"
    res["decode_many_max_abs_diff_vs_per_clip"] = max(float((wavs[k] - dwav[k]).abs().max()) for k, _ in base)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
