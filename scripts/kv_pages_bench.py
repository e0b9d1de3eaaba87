"""Ring decode attention alone, paged against contiguous: B = 32 streams, each querying a full ring of 2047 keys
(context 2048), for the 7B MHA shape (32 heads of 128) and a 3B GQA shape (24 query heads over 8 KV groups of 128).
The paged pool holds each stream's ring in pages of lm.KV_PAGE positions assigned in a scrambled order.  Device events
around many launches, the two forms alternated; the outputs are checked bit for bit.  Prints one JSON line with the
card's name and power limit.

usage: python scripts/kv_pages_bench.py [--launches 500] [--rounds 3] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rstnet_b200 import _lib, ops            # noqa: E402
from rstnet_b200.lm import KV_PAGE           # noqa: E402

SHAPES = {"7B MHA": (32, 32, 128), "3B GQA": (24, 8, 128)}   # (query heads, KV groups, head size)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kv_pages_bench.py measures on the GPU; no CUDA device found")
    dev, bf = torch.device("cuda", 0), torch.bfloat16
    lib, st = _lib.lib(), ops._stream()
    B, cap = 32, 2048
    log2 = KV_PAGE.bit_length() - 1
    stride = cap // KV_PAGE
    res = {"gpu": torch.cuda.get_device_name(dev), "B": B, "keys": cap - 1, "page": KV_PAGE, "shapes": {}}
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        res["power_limit"] = f"unknown ({e})"
    g = torch.Generator(device="cpu").manual_seed(0)
    for name, (nh, nkv, hs) in SHAPES.items():
        kv = torch.randn(2, B, nkv, cap, hs, generator=g).to(dev, bf)
        n_pages = B * stride
        table = torch.randperm(n_pages, generator=g).view(B, stride).to(torch.int32)
        pool = torch.empty(n_pages, 2, nkv, KV_PAGE, hs, dtype=bf, device=dev)
        pool[table.flatten().long().to(dev)] = kv.view(2, B, nkv, stride, KV_PAGE, hs).permute(1, 3, 0, 2, 4, 5).reshape(
            n_pages, 2, nkv, KV_PAGE, hs)
        pt = table.to(dev)
        q = torch.randn(B, nh * hs, generator=g).to(dev, bf)
        offset = torch.full((B,), 2 * cap + cap - 2, dtype=torch.int64, device=dev)   # wrapped; cap - 1 keys attendable
        outs = {k: torch.empty(B, nh * hs, dtype=bf, device=dev) for k in ("contiguous", "paged")}

        def launch(form):
            if form == "paged":
                _lib.check(lib.rstnet_lm_paged_decode_attention_bf16(q.data_ptr(), pool.data_ptr(), offset.data_ptr(), 1, None, None,
                                                                     outs[form].data_ptr(), B, B, nh, nkv, hs, cap, cap, pt.data_ptr(),
                                                                     stride, log2, st))
            else:
                _lib.check(lib.rstnet_lm_ring_decode_attention_bf16(q.data_ptr(), kv.data_ptr(), offset.data_ptr(), 1, None, None,
                                                                    outs[form].data_ptr(), B, B, nh, nkv, hs, cap, cap, st))

        times = {"contiguous": [], "paged": []}
        for form in times:
            for _ in range(20):
                launch(form)
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for form in times:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.launches):
                    launch(form)
                e1.record()
                torch.cuda.synchronize()
                times[form].append(1e3 * e0.elapsed_time(e1) / args.launches)
        same = torch.equal(outs["contiguous"].view(torch.int16), outs["paged"].view(torch.int16))
        kv_bytes = 2 * B * nkv * (cap - 1) * hs * 2
        c, p = min(times["contiguous"]), min(times["paged"])
        res["shapes"][name] = {"heads": nh, "kv_groups": nkv, "head_size": hs, "contiguous_us": times["contiguous"],
                               "paged_us": times["paged"], "paged_overhead": p / c - 1.0, "bit_identical": same,
                               "contiguous_kv_GBps": kv_bytes / c * 1e-3, "paged_kv_GBps": kv_bytes / p * 1e-3}
        del kv, pool
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
