"""Best-of-N TTS at 7B shapes (random init, bf16; the model and corpus of scripts/tts_batch.py).  Prints one JSON line:

  * best_of: InferenceImp.generate_many(n_samples=N) over the corpus -- one prompt prefill per utterance, forked into N
    rows that share its KV pages, each candidate's log-probability summed inside the frame graph;
  * separate: the same N x utterances listed one by one with sample_seed(seed, i) seeds (N prefills, N private copies of
    each prompt's KV), then a teacher-forced InferenceImp.score_many rescoring of every candidate to rank them;
  * for both: wall time, candidate frames/s (generated frames of all candidates over the wall time), peak KV pages held;
    best_of also checks that its candidates' codes equal the separate run's;
  * logprob_cost: device time per frame of the frame graph with logprob=True against the plain graph, every row active,
    alternating blocks of frames.

usage: python scripts/tts_best_of.py [--utts 16] [--n 4] [--capacity 32] [--seed 0] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rstnet_b200.infer import InferenceImp, sample_seed   # noqa: E402
from rstnet_b200.lm import KV_PAGE, Sampling   # noqa: E402
from tts_batch import corpus, gpt7b   # noqa: E402


class PagePeak:
    """the most KV pages held after any frame of a generate_many run"""

    def __init__(self, m):
        self.m, self.peak, self.orig = m, 0, m.forward_step

    def __enter__(self):
        def counted(*a, **kw):
            out = self.orig(*a, **kw)
            self.peak = max(self.peak, self.m._state.pages.in_use)
            return out
        self.m.forward_step = counted
        return self

    def __exit__(self, *a):
        del self.m.forward_step


def best_of(imp, items, n, cap, seeds):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with PagePeak(imp.model) as pk:
        out = {u: c for u, c in imp.generate_many(((u, s.cuda()) for u, s in items), cap, seeds=seeds, n_samples=n)}
    torch.cuda.synchronize()
    return out, time.perf_counter() - t0, pk.peak


def separate(imp, items, n, cap, seeds):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    listed = [((u, i), s) for u, s in items for i in range(n)]
    keys = {(u, i): sample_seed(seeds[u], i) for u, _ in items for i in range(n)}
    with PagePeak(imp.model) as pk:
        gen = {k: (c, raw) for k, c, raw in imp.generate_many(((k, s.cuda()) for k, s in listed), cap, seeds=keys, return_frames=True)}
    torch.cuda.synchronize()
    t_gen = time.perf_counter() - t0
    P = {u: imp._layout(s)[0] for u, s in items}
    src = dict(items)

    def scored():
        for (u, i), (_, raw) in gen.items():
            seq = torch.cat([src[u][:, :P[u]], raw.cpu().t()], 1)
            mask = torch.zeros(seq.shape, dtype=torch.float32)
            mask[:, P[u]:] = 1
            yield (u, i), seq, mask
    loss = {k: met["loss_audio"] for k, met in imp.score_many(scored(), capacity=cap)}
    torch.cuda.synchronize()
    return gen, loss, t_gen, time.perf_counter() - t0, pk.peak


def logprob_cost(m, cap, frames=40, blocks=3):
    dev = m.device
    sp = [Sampling()] * cap
    with m.streaming(cap, kv_pages=cap * -(-m.config.context // KV_PAGE)):
        m.reserve_kv(list(range(cap)), m.config.context)
        cur = torch.randint(0, 2048, (cap, 9, 1), device=dev)
        valid = torch.full((cap, 8), 2048, dtype=torch.int32, device=dev)
        keys = torch.arange(cap)

        def run(lp, k):
            nonlocal cur
            for _ in range(k):
                toks = m.forward_step(cur, audio_valid=valid, sample_key=keys, depth_ring_quirk=False, sampling=sp, logprob=lp)
                cur = toks[:, :, None]
            m.reset_streaming()

        for lp in (False, True):
            run(lp, 3)                          # warm-up and capture of both graphs
        times = {False: [], True: []}
        for _ in range(blocks):
            for lp in (False, True):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(lp, frames)
                e1.record()
                torch.cuda.synchronize()
                times[lp].append(e0.elapsed_time(e1) / frames)
    return {"plain_ms_per_frame": min(times[False]), "logprob_ms_per_frame": min(times[True]),
            "all_plain": times[False], "all_logprob": times[True]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=16)
    ap.add_argument("--n", type=int, default=4)
    ap.add_argument("--capacity", type=int, default=32)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    m = gpt7b(dev)
    imp = InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")
    items = corpus(a.utts, a.seed)
    seeds = {u: 1000 + i for i, (u, _) in enumerate(items)}
    G = {u: imp._layout(s)[1] for u, s in items}
    cand_frames = a.n * sum(G.values())
    # warm-up: the graphs of both paths on two utterances
    best_of(imp, items[:2], a.n, a.capacity, seeds)
    separate(imp, items[:1], a.n, a.capacity, seeds)
    bo, t_bo, peak_bo = best_of(imp, items, a.n, a.capacity, seeds)
    gen, loss, t_gen, t_sep, peak_sep = separate(imp, items, a.n, a.capacity, seeds)
    same = all(torch.equal(c.codes.cpu(), gen[(u, c.index)][0].cpu()) for u, cs in bo.items() for c in cs)
    # do the two rankings pick the same candidate? (the in-frame sums are the generation path's bf16 logits, the
    # rescoring the teacher-forced pass's)
    agree = sum(cs[0].index == min(range(a.n), key=lambda i: (loss[(u, i)], i)) for u, cs in bo.items())
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "utts": a.utts, "n_samples": a.n, "capacity": a.capacity, "candidate_frames": cand_frames,
           "best_of": {"seconds": t_bo, "candidate_frames_per_s": cand_frames / t_bo, "peak_pages": peak_bo},
           "separate": {"seconds": t_sep, "generate_seconds": t_gen, "rescore_seconds": t_sep - t_gen,
                        "candidate_frames_per_s": cand_frames / t_sep, "peak_pages": peak_sep},
           "codes_equal": same, "best_pick_agrees": f"{agree}/{len(bo)}",
           "logprob_cost": logprob_cost(m, a.capacity)}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
