"""Generation beyond fixed-length TTS at 7B shapes (random init, bf16; the model of scripts/tts_batch.py).  Prints one JSON
line with, per run, frames/s of generated frames, decode steps, row occupancy (generated frames / (steps x capacity)) and
the mean time per decode step:

  * fixed: the fixed-length TTS corpus of scripts/tts_batch.py at each capacity (host-built candidate tables, no status
    read), run --repeats times alternating with
  * windowed: the same corpus with lengths = (G - 2, G), so every row runs with the device's generation window and the
    host reads each frame's statuses one frame late (rows rarely stop one or two frames early);
  * asr / audio_only: corpora of those tasks with ragged lengths (ASR rows stop early when their stop rule fires).

usage: python scripts/gen_tasks_bench.py [--utts 48] [--capacities 32,48] [--repeats 2] [--seed 0] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from tts_batch import corpus, gpt7b   # noqa: E402
from rstnet_b200.infer import InferenceImp   # noqa: E402

TEXT_EMPTY, TEXT_PAD, PAD = 128002, 128003, 2049


def task_corpus(task, n, seed):
    """ragged items: ASR 50..300 audio frames then 20..200 text frames; audio_only 100..800 audio frames"""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        a = int(torch.randint(50, 301, (1,), generator=g)) if task == "ASR" else int(torch.randint(100, 801, (1,), generator=g))
        b = int(torch.randint(20, 201, (1,), generator=g)) if task == "ASR" else 0
        seq = torch.randint(0, 2048, (9, a + b), generator=g)
        seq[0, :a] = TEXT_EMPTY
        if task == "ASR":
            seq[0, a:] = torch.randint(0, 128000, (b,), generator=g)
            seq[1:, a:] = PAD
        out.append((f"{task}{i:04d}", seq))
    return out


def run(imp, items, cap, **kw):
    stats = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for out in imp.generate_many(((u, s.cuda()) for u, s in items), cap, stats=stats, **kw):
        n += 1
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    assert n == len(items)
    return {"frames_per_s": round(stats["row_frames"] / dt, 1), "steps": stats["frames"],
            "occupancy": round(stats["row_frames"] / (stats["frames"] * cap), 4),
            "ms_per_step": round(1e3 * dt / stats["frames"], 3), "seconds": round(dt, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=48)
    ap.add_argument("--capacities", default="32,48")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gen_tasks_bench measures on a GPU")
    m = gpt7b("cuda")
    m.use_cuda_graphs = True
    imp = InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")
    tts = corpus(a.utts, a.seed)
    lengths = {u: (int(s[0].eq(TEXT_EMPTY).sum()) - 2, int(s[0].eq(TEXT_EMPTY).sum())) for u, s in tts}
    caps = [int(c) for c in a.capacities.split(",")]
    res = {"gpu": torch.cuda.get_device_name(0), "utts": a.utts, "runs": []}
    for cap in caps:
        run(imp, tts[:cap], cap)                                   # warm-up: graphs of both paths
        run(imp, tts[:cap], cap, lengths=lengths)
        for rep in range(a.repeats):                               # alternate the two paths
            res["runs"].append({"kind": "fixed", "capacity": cap, "repeat": rep, **run(imp, tts, cap)})
            res["runs"].append({"kind": "windowed", "capacity": cap, "repeat": rep, **run(imp, tts, cap, lengths=lengths)})
        for task in ("ASR", "audio_only"):
            items = task_corpus(task, a.utts, a.seed + 1)
            res["runs"].append({"kind": task, "capacity": cap, **run(imp, items, cap, tasks={u: task for u, _ in items})})
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
