"""Teacher-forced scoring throughput of the Moshi twin (moshi.score_many), Moshi 7B shapes (MOSHI_7B of
scripts/moshi_duplex.py: context 3000) with random init in bf16, over a seeded ragged corpus (L uniform in 30..4000
frames, so some utterances run past the 3000-frame window; masks of ones).  Prints one JSON line:

  * scored frames/s of score_many at each capacity, and the mean chunk fill (real rows / launched rows);
  * the same corpus one utterance at a time through LMModel.forward + validate_model's two CrossEntropyAndAccuracy calls;
  * the card's name and power limit, read in the same call.

usage: python scripts/moshi_score_bench.py [--utts 64] [--capacities 4,8,16] [--seed 0] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from lm_score_bench import ChunkLog            # noqa: E402
from moshi_duplex import MOSHI_7B              # noqa: E402
from rstnet_b200.lm import CrossEntropyAndAccuracy   # noqa: E402
from rstnet_b200.moshi import AUDIO_WEIGHTS, LMModel, score_many   # noqa: E402


def corpus(n, seed, K):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        L = int(torch.randint(30, 4001, (1,), generator=g))
        seq = torch.randint(0, 2048, (K, L), generator=g)
        seq[0] = torch.randint(0, 32000, (L,), generator=g)
        out.append((f"utt{i:04d}", seq, torch.ones(K, L)))
    return out


def run(lm, items, cap):
    with ChunkLog() as log:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = dict(score_many(lm, iter(items), capacity=cap))
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    return out, wall, log


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--capacities", default="4,8,16")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("moshi_score_bench.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    lm = LMModel(**MOSHI_7B, device=dev, dtype=torch.bfloat16).eval()
    K = lm.num_codebooks
    items = corpus(args.utts, args.seed, K)
    frames = sum(s.shape[1] for _, s, _ in items)
    res = {"model": "Moshi 7B shapes, random init, bf16, context 3000", "utterances": len(items), "frames": frames,
           "past_window": sum(s.shape[1] > lm.context for _, s, _ in items), "gpu": torch.cuda.get_device_name(dev),
           "score_many": {}}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the numbers stay valid; the card's limit is then unknown
        res["power_limit"] = f"unknown ({e})"
    caps = [int(c) for c in args.capacities.split(",")]
    results = {}
    for cap in caps:
        run(lm, items[:2 * cap], cap)                       # warm-up: plans and chunk states of every width
        out, wall, log = run(lm, items, cap)
        results[cap] = out
        res["score_many"][str(cap)] = {"seconds": wall, "frames_per_s": frames / wall, "chunks": len(log.chunks),
                                       "mean_chunk_fill": log.fill()}
    # one utterance at a time: LMModel.forward + validate_model's CrossEntropyAndAccuracy calls
    s, k = items[0][1][None].to(dev), items[0][2][None].to(dev)
    lm(s, k)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    worst = 0.0
    for utt, seq, mask in items:
        s, k = seq[None].to(dev), mask[None].to(dev)
        audio, text = lm(s, k)
        la, _ = CrossEntropyAndAccuracy(audio, s[:, 1:9], k[:, 1:9], AUDIO_WEIGHTS, [2048] * 8)
        lt, _ = CrossEntropyAndAccuracy(text.unsqueeze(2), s[:, 0].unsqueeze(1), k[:, 0:1], [1], [32000])
        for key, v in (("loss_audio", la), ("loss_text", lt)):
            ref = results[caps[-1]][utt][key]
            worst = max(worst, abs(float(v) - ref) / abs(ref))
        del audio, text
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res["per_utterance_forward"] = {"seconds": wall, "frames_per_s": frames / wall,
                                    "max_rel_loss_diff_vs_score_many": worst}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
