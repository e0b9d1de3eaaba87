"""Duplex serving on paged KV: Moshi 7B shapes (as scripts/moshi_duplex.py: dim 4096, 32 layers, context 3000) through
`FrameScheduler` + `MoshiDuplexEngine(kv_pages=N)`, or with --gpt the GPT 7B `DuplexEngine` (context 2048).

Sessions are given seeded ages: each row is fast-forwarded to the position its age reaches at 12.5 frames/s (a KV ring
holds the last `context` of them), with pages reserved to match.  The ages of a population are drawn
uniformly from --age-min .. --age-max seconds (seeded; population B is the first B draws).  Seeded random bf16 weights.
Reports, after the card's name and power limit:

  overhead  the same B = --overhead-b population, contiguous rings against paged, alternated (--rounds each, a new
            engine per round): tick p50 / p99, and whether the tokens of the first ticks are identical;
  capacity  a fixed KV budget, the memory the largest contiguous B would use (free memory after the weights, less 3 GB,
            in whole rings): for each B, the pages the population holds at the end of its ticks, whether it fits, tick
            p50 / p99 where it fits, and the largest B with tick p99 < 80 ms;
  churn     a seeded arrival / departure trace through FrameScheduler(kv_headroom=H) on that budget: an initial
            population admitted (fast-forwarded) until the pool refuses, then Poisson arrivals of new sessions, and
            departures when a session reaches its drawn length; admissions, refusals (batch full / KV pool short),
            evictions, departures, tick p50/p99.

Everything is printed as JSON lines and, with --out FILE, written there as one JSON document.

    python scripts/duplex_kv_pages.py [--gpt] [--batches 40,48,...] [--ticks 40] [--out FILE]
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
from rstnet_b200.lm import KV_PAGE, GPT, Config, kv_page_bytes  # noqa: E402
from rstnet_b200.moshi import LMGen, LMModel  # noqa: E402
from rstnet_b200.serve import FRAME_SAMPLES, DuplexEngine, FrameScheduler, MoshiDuplexEngine  # noqa: E402
from specs import mimi_spec as S  # noqa: E402

DEV, BF = "cuda", torch.bfloat16
FPS = 12.5
BUDGET_MS = 80.0
MOSHI_7B = dict(dim=4096, text_card=32000, existing_text_padding_id=3, n_q=16, dep_q=8, card=2048, num_heads=32, num_layers=32,
                hidden_scale=4.125, causal=True, layer_scale=None, context=3000, max_period=10000, gating="silu",
                norm="rms_norm_f32", positional_embedding="rope", depformer_dim=1024, depformer_dim_feedforward=int(4.125 * 1024),
                depformer_num_heads=16, depformer_num_layers=6, depformer_causal=True, depformer_layer_scale=None,
                depformer_multi_linear=True, depformer_context=8, depformer_max_period=10000, depformer_gating="silu",
                depformer_pos_emb="none", depformer_weights_per_step=True,
                delays=[0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1])
GPT_7B = dict(block_size=4096, n_layer=32, n_embd=4096, n_head=32, head_size=128, intermediate_size=11008, padded_vocab_size=152064,
              audio_card=2050, n_q=8, dep_q=8, codecformer_dim=1024, codecformer_heads=16, codecformer_layers=6,
              codecformer_dim_feedforward=4224, context=2048)


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    line = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else ""
    name, power = ([s.strip() for s in line.split(",")] + ["?", "?"])[:2]
    return {"name": name or torch.cuda.get_device_name(0), "power_limit": power}


class Setup:
    """The model, the codec and how an engine over them is built and fast-forwarded."""

    def __init__(self, use_gpt: bool):
        torch.manual_seed(0)
        self.gpt = use_gpt
        self.lm = (GPT(Config(**GPT_7B), device=DEV, dtype=BF) if use_gpt else LMModel(**MOSHI_7B, device=DEV, dtype=BF)).eval()
        codec = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
        codec.load_state_dict(S.synthetic_weights(S.OFFICIAL, seed=41), strict=True)
        self.codec = codec.to(DEV).eval()
        c = self.lm.config
        self.context = c.context
        self.ring_bytes = c.n_layer * 2 * c.n_query_groups * c.context * c.head_size * 2
        self.page_bytes = kv_page_bytes(c)
        self.ring_pages = -(-c.context // KV_PAGE)

    def engine(self, B: int, kv_pages):
        kw = {} if kv_pages is None else dict(kv_pages=kv_pages)
        if self.gpt:
            return DuplexEngine(self.codec, self.lm, B, **kw)
        return MoshiDuplexEngine(self.codec, LMGen(self.lm), B, **kw)

    def drop(self):
        self.codec._stream_state = None
        self.lm._state = None
        gc.collect()
        torch.cuda.empty_cache()

    def pages_for(self, pos: int) -> int:
        return -(-min(int(pos), self.context) // KV_PAGE)

    def fast_forward(self, eng, rows, pos) -> None:
        """rows at positions pos (past the warm-up, a delay cache of valid ids), with pages reserved to match"""
        rows = [int(r) for r in rows]
        pos = np.asarray(pos, dtype=np.int64)
        st = self.lm._state
        idx = torch.tensor(rows, device=DEV)
        st.offset[idx] = torch.from_numpy(pos).to(DEV)
        st.pos_host[rows] = pos
        if not self.gpt:
            g = eng.lm_gen._st
            g.cache[idx] = 0
            g.off[idx] = torch.from_numpy(pos).to(DEV)
            g.off_host[rows] = pos
            g.valid[idx] = 1
        if eng.kv_pages is not None:
            self.lm.reserve_kv(rows, np.maximum(-(-pos // KV_PAGE), 1) * KV_PAGE)


AUDIO = None


def frame(s, t):
    i = (hash(s) + t) % 8
    return AUDIO[i % AUDIO.shape[0], i * FRAME_SAMPLES:(i + 1) * FRAME_SAMPLES]


def run_ticks(sch, ticks: int, warm: int = 5, keep_tokens: int = 0):
    """push a frame for every session and tick; -> tick times (ms, after `warm`), tokens of the first ticks, evictions"""
    lat, toks, ev = [], [], 0
    for t in range(warm + ticks):
        for s in sch.sessions():
            sch.push(s, frame(s, t))
        t0 = time.perf_counter()
        out = sch.tick()
        dt = 1e3 * (time.perf_counter() - t0)
        ev += len(sch.take_evicted())
        if t >= warm:
            lat.append(dt)
        if t < keep_tokens:
            toks.append({s: None if v[0] is None else v[0].clone() for s, v in out.items()})
    return lat, toks, ev


def stats(lat) -> dict:
    return {"tick_ms_p50": float(np.percentile(lat, 50)), "tick_ms_p99": float(np.percentile(lat, 99)),
            "tick_ms_max": float(np.max(lat)), "ticks": len(lat)}


def population(setup: Setup, B: int, ages) -> np.ndarray:
    return np.round(FPS * ages[:B]).astype(np.int64)


def overhead_part(setup: Setup, B: int, ages, ticks: int, rounds: int) -> dict:
    pos = population(setup, B, ages)
    pool = int(sum(setup.pages_for(p + ticks + 10) for p in pos))
    lat = {"contiguous": [], "paged": []}
    toks = {}
    for _ in range(rounds):
        for name, kv in (("contiguous", None), ("paged", pool)):
            eng = setup.engine(B, kv)
            sch = FrameScheduler(eng, B)
            for s in range(B):
                sch.admit(s)
            setup.fast_forward(eng, range(B), pos)
            l, tk, ev = run_ticks(sch, ticks, keep_tokens=10)
            assert ev == 0
            lat[name] += l
            toks.setdefault(name, tk)
            del sch, eng
            setup.drop()
    same = all(set(a) == set(b) and all((a[s] is None and b[s] is None) or torch.equal(a[s], b[s]) for s in a)
               for a, b in zip(toks["contiguous"], toks["paged"]))
    return {"B": B, "pool_pages": pool, "rounds": rounds, "contiguous": stats(lat["contiguous"]), "paged": stats(lat["paged"]),
            "tokens_identical_first_10_ticks": bool(same)}


def capacity_part(setup: Setup, n_pages: int, batches, ages, ticks: int) -> list:
    out = []
    for B in batches:
        pos = population(setup, B, ages)
        need = int(sum(setup.pages_for(p + ticks + 5) for p in pos))
        r = {"B": B, "pages_at_start": int(sum(setup.pages_for(p) for p in pos)), "pages_at_end": need,
             "pool_pages": n_pages, "fits": need <= n_pages}
        if r["fits"]:
            try:
                eng = setup.engine(B, n_pages)
                sch = FrameScheduler(eng, B)
                for s in range(B):
                    sch.admit(s)
                setup.fast_forward(eng, range(B), pos)
                lat, _, ev = run_ticks(sch, ticks)
                r.update(stats(lat), evicted=ev, pages_in_use=n_pages - eng.kv_pages_free)
                del sch, eng
            except torch.cuda.OutOfMemoryError:
                r["oom"] = True
            setup.drop()
        print(json.dumps({"capacity": r}), flush=True)
        out.append(r)
    return out


def churn_part(setup: Setup, n_pages: int, rows: int, headroom: int, ticks: int, rate: float, age_min: float, age_max: float,
               seed: int) -> dict:
    rng = np.random.default_rng(seed)
    eng = setup.engine(rows, n_pages)
    sch = FrameScheduler(eng, rows, kv_headroom=headroom)
    length, started = {}, {}
    nxt = 0
    res = {"rows": rows, "pool_pages": n_pages, "kv_headroom": headroom, "arrival_rate_per_tick": rate, "ticks": ticks,
           "initial": 0, "admitted": 0, "refused_batch_full": 0, "refused_kv_pool": 0, "evicted": 0, "departed": 0}
    # initial population: sessions part-way through their drawn lengths, admitted while the pool takes them
    while len(sch.sessions()) < rows:
        L = int(round(FPS * rng.uniform(age_min, age_max)))
        p = int(rng.integers(0, L))
        if eng.kv_pages_free < setup.pages_for(p) + headroom + 1:
            break
        row = sch.admit(nxt)
        setup.fast_forward(eng, [row], [p])
        length[nxt], started[nxt] = L, -p
        nxt += 1
    res["initial"] = len(sch.sessions())
    lat, conc = [], []
    for t in range(ticks):
        for s in [s for s in sch.sessions() if t - started[s] >= length[s]]:
            sch.release(s)
            res["departed"] += 1
        for _ in range(rng.poisson(rate)):
            try:
                sch.admit(nxt)
                length[nxt], started[nxt] = int(round(FPS * rng.uniform(age_min, age_max))), t
                res["admitted"] += 1
            except RuntimeError:
                res["refused_batch_full" if sch.free_rows() == 0 else "refused_kv_pool"] += 1
            nxt += 1
        for s in sch.sessions():
            sch.push(s, frame(s, t))
        conc.append(len(sch.sessions()))
        t0 = time.perf_counter()
        sch.tick()
        lat.append(1e3 * (time.perf_counter() - t0))
        res["evicted"] += len(sch.take_evicted())
    res.update(stats(lat[5:]), sessions_min=int(min(conc)), sessions_max=int(max(conc)),
               pages_free_at_end=int(eng.kv_pages_free))
    del sch, eng
    setup.drop()
    return res


def main():
    global AUDIO
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpt", action="store_true", help="the GPT 7B DuplexEngine (context 2048) instead of Moshi 7B")
    ap.add_argument("--batches", default="40,48,56,64,80,96,128,160,192,256")
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--overhead-b", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--age-min", type=float, default=10.0)
    ap.add_argument("--age-max", type=float, default=240.0)
    ap.add_argument("--churn-rows", type=int, default=128)
    ap.add_argument("--churn-ticks", type=int, default=300)
    ap.add_argument("--churn-rate", type=float, default=0.3, help="mean arrivals per tick")
    ap.add_argument("--kv-headroom", type=int, default=8)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--skip", default="", help="comma list of parts to skip: overhead, capacity, churn")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("duplex_kv_pages.py measures on a CUDA device; none is visible")
    res = {"card": card(), "model": ("gpt-7b shapes (context 2048)" if a.gpt else "moshi-7b shapes (context 3000)")
           + ", random bf16 weights", "page": KV_PAGE,
           "ages": f"session ages uniform over {a.age_min:g}-{a.age_max:g} s (seed {a.seed}), 12.5 positions per second"}
    print(json.dumps(res), flush=True)
    setup = Setup(a.gpt)
    AUDIO = S.synthetic_audio(4, FRAME_SAMPLES * 8, seed=3)[:, 0]
    ages = np.random.default_rng(a.seed).uniform(a.age_min, a.age_max, 256)
    skip = set(a.skip.split(","))
    res.update(ring_gb=setup.ring_bytes / 1e9, page_mib=setup.page_bytes / 2 ** 20, ring_pages=setup.ring_pages)
    if "overhead" not in skip:
        res["overhead"] = overhead_part(setup, a.overhead_b, ages, a.ticks, a.rounds)
        print(json.dumps({"overhead": res["overhead"]}), flush=True)
    setup.drop()
    free, _ = torch.cuda.mem_get_info()
    b_max = int((free - 3e9) // setup.ring_bytes)
    n_pages = b_max * setup.ring_bytes // setup.page_bytes
    res["budget"] = {"largest_contiguous_B": b_max, "kv_gb": b_max * setup.ring_bytes / 1e9, "pool_pages": int(n_pages)}
    print(json.dumps({"budget": res["budget"]}), flush=True)
    if "capacity" not in skip:
        res["capacity"] = capacity_part(setup, n_pages, [int(b) for b in a.batches.split(",")], ages, a.ticks)
        ok = [r["B"] for r in res["capacity"] if r.get("fits") and "tick_ms_p99" in r and r["tick_ms_p99"] < BUDGET_MS]
        res["largest_B_p99_under_80ms"] = max(ok) if ok else None
    if "churn" not in skip:
        res["churn"] = churn_part(setup, n_pages, a.churn_rows, a.kv_headroom, a.churn_ticks, a.churn_rate, a.age_min, a.age_max,
                                  a.seed + 1)
        print(json.dumps({"churn": res["churn"]}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
