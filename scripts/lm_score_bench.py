"""Teacher-forced scoring throughput (InferenceImp.score_many), 7B shapes with random init in bf16, context 2048, over a
seeded ragged corpus (L uniform in 30..1000 frames, masks of ones).  Prints one JSON line:

  * scored frames/s of score_many at each capacity, and the mean chunk fill (real rows / launched rows);
  * the same corpus one utterance at a time through GPT.forward + CrossEntropyAndAccuracy (audio and text);
  * the cross-entropy launches' share of score_many's time (device events around each eager launch pair, in a run of
    its own) and their achieved bandwidth (bytes of the logit rows they read) against the 3.35 TB/s data-sheet figure;
  * the card's name and power limit, read in the same call.

usage: python scripts/lm_score_bench.py [--utts 64] [--capacities 4,8,16] [--seed 0] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rstnet_b200 import lm                      # noqa: E402
from rstnet_b200.infer import InferenceImp      # noqa: E402
from rstnet_b200.lm import GPT, Config, CrossEntropyAndAccuracy   # noqa: E402

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def gpt7b(dev):
    cfg = Config(block_size=4096, n_layer=32, n_embd=4096, n_head=32, head_size=128, intermediate_size=11008,
                 padded_vocab_size=152064, audio_card=2050, n_q=8, dep_q=8, codecformer_dim=1024, codecformer_heads=16,
                 codecformer_layers=6, codecformer_dim_feedforward=4224, context=2048)
    return GPT(cfg, device=dev, dtype=torch.bfloat16).eval()


def corpus(n, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        L = int(torch.randint(30, 1001, (1,), generator=g))
        seq = torch.randint(0, 2048, (9, L), generator=g)
        seq[0] = torch.randint(0, 128000, (L,), generator=g)
        out.append((f"utt{i:04d}", seq, torch.ones(9, L)))
    return out


class ChunkLog:
    """Rows of every scoring chunk (real rows, launched width) and, with events=True, device time of every
    cross-entropy call."""

    def __init__(self, events=False):
        self.chunks, self.ce, self.events = [], [], events

    def __enter__(self):
        orig_chunk, orig_ce = lm._LMState.row_chunk, lm.cross_entropy_sums
        log = self

        def row_chunk(st, todo, head=False):
            ch, segs = orig_chunk(st, todo, head)
            log.chunks.append((sum(s[3] for s in segs), ch.M))
            return ch, segs

        def ce(logits, *a, **kw):
            if not log.events:
                return orig_ce(logits, *a, **kw)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = orig_ce(logits, *a, **kw)
            e1.record()
            log.ce.append((e0, e1, logits.shape[1]))
            return r

        self._orig = (orig_chunk, orig_ce)
        lm._LMState.row_chunk, lm.cross_entropy_sums = row_chunk, ce
        return self

    def __exit__(self, *a):
        lm._LMState.row_chunk, lm.cross_entropy_sums = self._orig

    def fill(self):
        return sum(n for n, _ in self.chunks) / max(1, sum(M for _, M in self.chunks))

    def ce_stats(self, dep_q):
        """(seconds, bytes read): calls alternate text / audio per chunk; padding rows are not read."""
        t = sum(a.elapsed_time(b) for a, b, _ in self.ce) * 1e-3
        nbytes = 0
        for i, (_, _, V) in enumerate(self.ce):
            n = self.chunks[i // 2][0]
            nbytes += 2 * V * n * (1 if i % 2 == 0 else dep_q)
        return t, nbytes


def run(imp, items, cap, events=False):
    with ChunkLog(events) as log:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = dict(imp.score_many(iter(items), capacity=cap))
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
        raise SystemExit("lm_score_bench.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    m = gpt7b(dev)
    imp = InferenceImp(None, m, "teacher-force", 0.7, 25, 0.8, 30, "TTS")
    items = corpus(args.utts, args.seed)
    frames = sum(s.shape[1] for _, s, _ in items)
    res = {"model": "7B shapes, random init, bf16, context 2048", "utterances": len(items), "frames": frames,
           "gpu": torch.cuda.get_device_name(dev), "score_many": {}}
    try:
        import subprocess
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the numbers stay valid; the card's limit is then unknown
        res["power_limit"] = f"unknown ({e})"
    caps = [int(c) for c in args.capacities.split(",")]
    for cap in caps:
        run(imp, items[:2 * cap], cap)                      # warm-up: plans and chunk states of every width
        out, wall, log = run(imp, items, cap)
        res["score_many"][str(cap)] = {"seconds": wall, "frames_per_s": frames / wall, "chunks": len(log.chunks),
                                       "mean_chunk_fill": log.fill()}
    # the cross-entropy launches' share, eager events around each call, in a run of its own
    cap = caps[-1]
    _, wall, log = run(imp, items, cap, events=True)
    t_ce, nbytes = log.ce_stats(m.config.dep_q)
    res["cross_entropy"] = {"capacity": cap, "seconds": t_ce, "share_of_score_many": t_ce / wall, "bytes": nbytes,
                            "GB_per_s": nbytes / t_ce / 1e9, "share_of_3.35TB_per_s": nbytes / t_ce / HBM_PEAK,
                            "note": "event pairs around each eager call: include host-enqueue gaps between its two launches"}
    # the kernel alone on a full chunk's rows, back to back (no host gaps): text 128 x 152064, audio 1024 x 2050 (8 groups)
    g = torch.Generator(device=dev).manual_seed(1)
    res["cross_entropy_isolated"] = {}
    for name, rows, V, G in (("text", 128, m.config.padded_vocab_size, 1), ("audio", 128 * 8, m.config.audio_card, 8)):
        x = torch.randn(rows, V, device=dev, generator=g).to(torch.bfloat16)
        y = torch.randint(0, V, (rows,), device=dev, generator=g)
        w = torch.ones(rows, device=dev)
        acc = torch.zeros(1, G, 5, dtype=torch.float64, device=dev)
        nll = torch.empty(rows, device=dev)
        pred = torch.empty(rows, dtype=torch.int32, device=dev)
        for _ in range(5):
            lm.cross_entropy_sums(x, y, w, G, acc=acc, nll=nll, pred=pred)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 200
        e0.record()
        for _ in range(n):
            lm.cross_entropy_sums(x, y, w, G, acc=acc, nll=nll, pred=pred)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / n
        res["cross_entropy_isolated"][name] = {"rows": rows, "V": V, "us_per_call": us, "GB_per_s": 2 * rows * V / us / 1e3,
                                               "share_of_3.35TB_per_s": 2 * rows * V / (us * 1e-6) / HBM_PEAK}
    # one utterance at a time: GPT.forward + CrossEntropyAndAccuracy (audio and text), as the reference's teacher force
    def serial(sub):
        for _, seq, mask in sub:
            s, mk = seq[None].to(dev), mask[None].to(dev)
            audio, text = m(s)
            CrossEntropyAndAccuracy(audio, s[:, 1:], mk[:, 1:], [1] * 8, [2049] * 8)
            CrossEntropyAndAccuracy(text.unsqueeze(2), s[:, 0].unsqueeze(1), mk[:, 0:1], [1], [128003])
    serial(items[:2])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    serial(items)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res["forward_one_at_a_time"] = {"seconds": wall, "frames_per_s": frames / wall}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
