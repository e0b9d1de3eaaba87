"""Batch TTS over a corpus of utterances with different prompt and generation lengths (InferenceImp.generate_many),
7B shapes with random init in bf16 (the model of bench.py's cfg4_infer).  Prints one JSON line:

  * frames/s and tokens/s (9 tokens per generated frame: text + 8 audio) of the whole corpus at each capacity;
  * row occupancy: generated frames / (decode steps x capacity);
  * the paged KV pool of each run (--kv-gb: a pool of floor(X * 2^30 / kv_page_bytes) pages shared by every capacity;
    without it each capacity gets a whole ring per row) and the frames run while an utterance waited for pages;
  * whether every capacity produced the same codes;
  * the share of the time spent in ragged prefill (GPT.prefill_streams), timed with device events;
  * the ceiling: uniform InferenceImp.generate at B = 32 (every row the same layout, as cfg4_infer);
  * the serial rate: InferenceImp.generate at B = 1 on a few utterances, extrapolated to the corpus.

usage: python scripts/tts_batch.py [--utts 256] [--capacities 32,48] [--kv-gb X] [--seed 0] [--no-baselines] [--out FILE]
"""
import argparse
import hashlib
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rstnet_b200.infer import InferenceImp   # noqa: E402
from rstnet_b200.lm import GPT, KV_PAGE, Config, kv_page_bytes, kv_pages_for_budget   # noqa: E402

TEXT_EMPTY = 128002


def gpt7b(dev):
    cfg = Config(block_size=4096, n_layer=32, n_embd=4096, n_head=32, head_size=128, intermediate_size=11008,
                 padded_vocab_size=152064, audio_card=2050, n_q=8, dep_q=8, codecformer_dim=1024, codecformer_heads=16,
                 codecformer_layers=6, codecformer_dim_feedforward=4224, context=2048)
    return GPT(cfg, device=dev, dtype=torch.bfloat16).eval()


def corpus(n, seed):
    """P uniform in 20..120 prompt frames, G uniform in 100..1000 frames to generate."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        P = int(torch.randint(20, 121, (1,), generator=g))
        G = int(torch.randint(100, 1001, (1,), generator=g))
        seq = torch.randint(0, 2048, (9, P + G), generator=g)
        seq[0, :P] = torch.randint(0, 128000, (P,), generator=g)
        seq[0, P:] = TEXT_EMPTY
        out.append((f"utt{i:04d}", seq))
    return out


class PrefillTimer:
    """Device time of every prefill_streams call (events around it, read after the run)."""

    def __init__(self, m):
        self.m, self.events, self.orig = m, [], m.prefill_streams

    def __enter__(self):
        def timed(prompts):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            self.orig(prompts)
            e1.record()
            self.events.append((e0, e1))
        self.m.prefill_streams = timed
        return self

    def __exit__(self, *a):
        del self.m.prefill_streams

    def seconds(self):
        return sum(a.elapsed_time(b) for a, b in self.events) * 1e-3


def run_many(imp, items, capacity, dev, kv_pages=None):
    m = imp.model
    steps = [0]
    orig = m.forward_step

    def counted(*a, **kw):
        steps[0] += 1
        return orig(*a, **kw)

    m.forward_step = counted
    try:
        with PrefillTimer(m) as pt:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            stats = {}
            out = dict(imp.generate_many(((u, s.to(dev)) for u, s in items), capacity, kv_pages=kv_pages, stats=stats))
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            prefill = pt.seconds()
    finally:
        del m.forward_step
    return out, wall, prefill, steps[0], stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=256)
    ap.add_argument("--capacities", default="32,48")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--serial-utts", type=int, default=3)
    ap.add_argument("--kv-gb", type=float, default=None, help="KV budget in GiB, the same paged pool at every capacity")
    ap.add_argument("--baselines", action=argparse.BooleanOptionalAction, default=True,
                    help="also time uniform generate at B = 32 and serial B = 1")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tts_batch.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda", 0)
    m = gpt7b(dev)
    imp = InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")
    items = corpus(args.utts, args.seed)
    frames = sum(int((s[0] == TEXT_EMPTY).sum()) for _, s in items)
    res = {"model": "7B shapes, random init, bf16, context 2048", "utterances": len(items), "generated_frames": frames,
           "gpu": torch.cuda.get_device_name(dev), "batched": {}, "kv_page_positions": KV_PAGE,
           "kv_page_bytes": kv_page_bytes(m.config), "kv_gb": args.kv_gb}
    try:
        import subprocess
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the number stays valid; the card's limit is then unknown
        res["power_limit"] = f"unknown ({e})"
    # warm-up (plans, chunk states, the frame graph of each width) on the corpus' prompts with 8 frames to generate
    warm = [(u, s[:, :s.shape[1] - int((s[0] == TEXT_EMPTY).sum()) + 8]) for u, s in items]
    pool = None if args.kv_gb is None else kv_pages_for_budget(m.config, args.kv_gb)
    digests = set()
    for cap in [int(c) for c in args.capacities.split(",")]:
        run_many(imp, warm[:2 * cap], cap, dev, pool)
        out, wall, prefill, steps, stats = run_many(imp, items, cap, dev, pool)
        digest = hashlib.sha256(b"".join(out[u].cpu().numpy().tobytes() for u, _ in items)).hexdigest()
        digests.add(digest)
        res["batched"][str(cap)] = {"seconds": wall, "frames_per_s": frames / wall, "tokens_per_s": 9 * frames / wall,
                                    "decode_steps": steps, "row_occupancy": frames / (steps * cap),
                                    "prefill_share": prefill / wall, "wait_frames": stats["wait_frames"],
                                    "kv_pages": pool if pool is not None else cap * -(-m.config.context // KV_PAGE),
                                    "codes_sha256": digest}
        del out
        torch.cuda.empty_cache()
    res["codes_identical_across_capacities"] = len(digests) == 1
    if not args.baselines:
        return finish(res, args.out)
    # ceiling: every row the same layout (cfg4_infer's shape), B = 32
    P, G, B = 70, 550, 32
    seq = items[0][1][:, :P + G].clone()
    seq[0, P:] = TEXT_EMPTY
    seq[0, :P] = items[0][1][0, :P]
    batch = seq.unsqueeze(0).expand(B, -1, -1).contiguous().to(dev)
    imp.generate(batch[:, :, :P + 8])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    imp.generate(batch)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res["uniform_generate_B32"] = {"prompt": P, "generated": G, "frames_per_s": B * G / wall, "tokens_per_s": 9 * B * G / wall}
    # serial: B = 1 on a few utterances, extrapolated to the corpus by frames
    sub = items[:args.serial_utts]
    imp.generate(sub[0][1][None, :, :sub[0][1].shape[1] - int((sub[0][1][0] == TEXT_EMPTY).sum()) + 4].to(dev))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sub_frames = 0
    for _, s in sub:
        imp.generate(s[None].to(dev))
        sub_frames += int((s[0] == TEXT_EMPTY).sum())
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    res["serial_B1_extrapolated"] = {"measured_utterances": len(sub), "frames_per_s": sub_frames / wall,
                                     "tokens_per_s": 9 * sub_frames / wall, "corpus_seconds_extrapolated": frames / (sub_frames / wall)}
    finish(res, args.out)


def finish(res, out):
    line = json.dumps(res)
    print(line)
    if out:
        with open(out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
