"""Session suspend / resume at 7B shapes (random bf16 weights): the GPT 7B `DuplexEngine` on paged KV (context 2048), or
with --moshi the Moshi 7B `MoshiDuplexEngine` (context 3000), set up as scripts/duplex_kv_pages.py does.

Reports, after the card's name and power limit:

  cost    one session suspended and resumed (into another row) against its age (--ages seconds): the blob's bytes,
          the KV pages it held, and the suspend (table + gather) / resume (table + scatter) time, synchronised, with the
          rate through the host link; the blob comes from a pool pinned beforehand (`pin_host_blobs`);
  live    a B = --live-b batch ticking while one session per tick is suspended and the one suspended on the previous
          tick resumed, at each --ctas value, alternated with ticks without swaps in the same run: tick p50 / p99;
  churn   the churn trace of scripts/duplex_kv_pages.py (--churn-rows rows, the same arrivals) through
          FrameScheduler(on_short="suspend"), with --pin-blobs whole-ring blobs pinned beforehand: evictions,
          suspensions, resumes, the mean and worst lag of the suspended sessions, tick p50 / p99.

    python scripts/duplex_suspend.py [--moshi] [--skip cost,live,churn] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import duplex_kv_pages as K  # noqa: E402
from rstnet_b200.lm import KV_PAGE  # noqa: E402
from rstnet_b200.serve import FRAME_SAMPLES, FrameScheduler  # noqa: E402
from specs import mimi_spec as S  # noqa: E402

FPS = K.FPS


def cost_part(setup, ages, ctas: int) -> list:
    out = []
    pos = [int(round(FPS * a)) for a in ages]
    eng = setup.engine(4, 2 * max(setup.pages_for(p) for p in pos) + 4)
    eng.swap_ctas = ctas
    eng.reset_rows([0, 1], seed=1)
    eng.step({0: torch.zeros(eng.frame_samples), 1: torch.zeros(eng.frame_samples)}, [0, 1])   # builds every plan
    eng.release_rows([0, 1])
    eng.pin_host_blobs(1, eng.row_bytes(max(pos)))          # the suspends below allocate no pinned memory
    for age, p in zip(ages, pos):
        for rep in range(3):
            eng.reset_rows([0], seed=2)
            setup.fast_forward(eng, [0], [p])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            st = eng.suspend_rows([0])[0]
            st.ready.synchronize()
            t1 = time.perf_counter()
            eng.reclaim()
            eng.resume_rows([1], [st])
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            eng.release_rows([1])
        r = {"age_s": age, "positions": p, "pages": setup.pages_for(p), "nbytes": st.nbytes,
             "suspend_ms": 1e3 * (t1 - t0), "resume_ms": 1e3 * (t2 - t1),
             "suspend_gb_s": st.nbytes / (t1 - t0) / 1e9, "resume_gb_s": st.nbytes / (t2 - t1) / 1e9}
        print(json.dumps({"cost": r}), flush=True)
        out.append(r)
    del eng
    setup.drop()
    return out


def live_part(setup, B: int, ages, ticks: int, ctas_list) -> dict:
    pos = K.population(setup, B, ages)
    pool = int(sum(setup.pages_for(p + 3 * ticks + 40) for p in pos)) + 64
    eng = setup.engine(B + 1, pool)
    sch = FrameScheduler(eng, B + 1)
    for s in range(B):
        sch.admit(s, seed=s)
    setup.fast_forward(eng, range(B), pos)
    eng.pin_host_blobs(3, eng.row_bytes(int(pos.max()) + 3 * ticks + 40))
    res = {"B": B, "pool_pages": pool}
    t = 0

    def tick():
        nonlocal t
        for s in list(sch.sessions()) + sch.suspended():
            sch.push(s, K.frame(s, t))
        t0 = time.perf_counter()
        sch.tick()
        t += 1
        return 1e3 * (time.perf_counter() - t0)

    for _ in range(5):
        tick()
    lat = {"none": []}
    for c in ctas_list:
        lat[f"ctas_{c}"] = []
    for rnd in range(2):
        lat["none"] += [tick() for _ in range(ticks)]
        for c in ctas_list:
            eng.swap_ctas = c
            prev = None
            for i in range(ticks):
                s = i % B
                if s in sch.sessions():
                    sch.suspend(s)
                if prev is not None:
                    sch.resume(prev)
                prev = s
                lat[f"ctas_{c}"].append(tick())
            if prev is not None:
                sch.resume(prev)
            lat["none"] += [tick() for _ in range(ticks)]
    for k, v in lat.items():
        res[k] = K.stats(v)
    del sch, eng
    setup.drop()
    return res


def churn_part(setup, n_pages: int, rows: int, headroom: int, ticks: int, rate: float, age_min: float, age_max: float, seed: int,
               pin_blobs: int):
    rng = np.random.default_rng(seed)
    eng = setup.engine(rows, n_pages)
    eng.pin_host_blobs(pin_blobs, eng.row_bytes(setup.context))    # suspension allocates nothing while serving
    sch = FrameScheduler(eng, rows, kv_headroom=headroom, on_short="suspend")
    length, started, done = {}, {}, {}
    nxt = 0
    res = {"rows": rows, "pool_pages": n_pages, "kv_headroom": headroom, "arrival_rate_per_tick": rate, "ticks": ticks,
           "initial": 0, "admitted": 0, "refused_batch_full": 0, "refused_kv_pool": 0, "evicted": 0, "departed": 0}
    while len(sch.sessions()) < rows:
        L = int(round(FPS * rng.uniform(age_min, age_max)))
        p = int(rng.integers(0, L))
        if eng.kv_pages_free < setup.pages_for(p) + headroom + 1:
            break
        row = sch.admit(nxt, seed=nxt)
        setup.fast_forward(eng, [row], [p])
        length[nxt], done[nxt] = L, p
        nxt += 1
    res["initial"] = len(sch.sessions())
    lat, conc, lag = [], [], {}
    for t in range(ticks):
        for s in [s for s in list(sch.sessions()) + sch.suspended() if done[s] >= length[s]]:
            if s in sch.lag:
                lag[s] = sch.lag[s]
            sch.release(s)
            res["departed"] += 1
        for _ in range(rng.poisson(rate)):
            try:
                sch.admit(nxt, seed=nxt)
                length[nxt], done[nxt] = int(round(FPS * rng.uniform(age_min, age_max))), 0
                res["admitted"] += 1
            except RuntimeError:
                res["refused_batch_full" if sch.free_rows() == 0 else "refused_kv_pool"] += 1
            nxt += 1
        for s in list(sch.sessions()) + sch.suspended():
            sch.push(s, K.frame(s, t))
        conc.append(len(sch.sessions()))
        t0 = time.perf_counter()
        for s in sch.tick():
            done[s] += 1
        lat.append(1e3 * (time.perf_counter() - t0))
        res["evicted"] += len(sch.take_evicted())
    lag.update({s: v for s, v in sch.lag.items() if s not in lag})
    for s in sch.suspended():                 # still suspended at the end: lagging by their time so far
        lag[s] = lag.get(s, 0) + ticks - sch._suspended_at[s]
    lags = [v for v in lag.values() if v > 0]
    res.update(K.stats(lat[5:]), suspensions=sch.suspensions, resumes=sch.resumes, suspended_at_end=len(sch.suspended()),
               lag_ticks_mean=float(np.mean(lags)) if lags else 0.0, lag_ticks_max=int(max(lags)) if lags else 0,
               sessions_min=int(min(conc)), sessions_max=int(max(conc)))
    del sch, eng
    setup.drop()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--moshi", action="store_true", help="the Moshi 7B MoshiDuplexEngine (context 3000) instead of GPT 7B")
    ap.add_argument("--ages", default="10,30,60,120,240")
    ap.add_argument("--cost-ctas", type=int, default=32)
    ap.add_argument("--live-b", type=int, default=32)
    ap.add_argument("--live-ticks", type=int, default=40)
    ap.add_argument("--ctas", default="8,32")
    ap.add_argument("--age-min", type=float, default=10.0)
    ap.add_argument("--age-max", type=float, default=240.0)
    ap.add_argument("--churn-rows", type=int, default=128)
    ap.add_argument("--churn-ticks", type=int, default=300)
    ap.add_argument("--churn-rate", type=float, default=0.3)
    ap.add_argument("--kv-headroom", type=int, default=8)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--pin-blobs", type=int, default=4, help="whole-ring blobs pinned up front for the churn's suspensions")
    ap.add_argument("--skip", default="")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("duplex_suspend.py measures on a CUDA device; none is visible")
    res = {"card": K.card(), "model": ("moshi-7b shapes (context 3000)" if a.moshi else "gpt-7b shapes (context 2048)")
           + ", random bf16 weights", "page": KV_PAGE}
    print(json.dumps(res), flush=True)
    setup = K.Setup(not a.moshi)
    K.AUDIO = S.synthetic_audio(4, FRAME_SAMPLES * 8, seed=3)[:, 0]
    ages = np.random.default_rng(a.seed).uniform(a.age_min, a.age_max, 256)
    skip = set(a.skip.split(","))
    if "cost" not in skip:
        res["cost"] = cost_part(setup, [float(x) for x in a.ages.split(",")], a.cost_ctas)
    if "live" not in skip:
        res["live"] = live_part(setup, a.live_b, ages, a.live_ticks, [int(c) for c in a.ctas.split(",")])
        print(json.dumps({"live": res["live"]}), flush=True)
    if "churn" not in skip:
        free, _ = torch.cuda.mem_get_info()
        b_max = int((free - 3e9) // setup.ring_bytes)
        n_pages = b_max * setup.ring_bytes // setup.page_bytes
        res["churn"] = churn_part(setup, int(n_pages), a.churn_rows, a.kv_headroom, a.churn_ticks, a.churn_rate, a.age_min,
                                  a.age_max, a.seed + 1, a.pin_blobs)
        print(json.dumps({"churn": res["churn"]}), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
