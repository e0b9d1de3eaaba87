"""Time the persistent depth-transformer kernel alone (7B shapes) and the pieces of an LM frame."""
import json
import sys

import torch

sys.path.insert(0, ".")
import bench

dev = torch.device("cuda", 0)
res = {}
m = bench._gpt7b(dev, context=2048)


def timeit(fn, n=30):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def one(B):
    with m.streaming(B):
        st = m._state
        st.tout.normal_()
        st.tokens.random_(0, 2048)
        for kv in st.kv:
            kv.normal_()
        st.offset.fill_(2100); st.pos_host[:] = 2100
        r = {}
        r["depth_8steps_sampled_ms"] = timeit(lambda: st._depth_frame(0, 8, True, True, 30, 0.8, [2048] * 8))
        r["depth_8steps_nosample_ms"] = timeit(lambda: st._depth_frame(0, 8, True, False))
        r["depth_1step_nosample_ms"] = timeit(lambda: st._depth_frame(0, 1, True, False))
        import os
        for dbg, nm in ((1, "no_mma"), (2, "no_loads"), (4, "no_epilogue"), (7, "barriers_only")):
            os.environ["RSTNET_DEPTH_DBG"] = str(dbg)
            r[f"depth_1step_{nm}_ms"] = timeit(lambda: st._depth_frame(0, 1, True, False))
        os.environ["RSTNET_DEPTH_DBG"] = "0"
        # per-phase stamps of CTA 0 for one step (k = 3)
        from rstnet_b200 import _lib
        tr = torch.zeros(1024, dtype=torch.int64, device=dev)
        _lib.lib().rstnet_lm_depth_frame_set_trace(st.df, tr.data_ptr())
        st._depth_frame(3, 4, True, True, 30, 0.8, [2048] * 8)
        torch.cuda.synchronize()
        _lib.lib().rstnet_lm_depth_frame_set_trace(st.df, None)
        t = tr.cpu().tolist()
        n = max(i for i, v in enumerate(t) if v) + 1
        d = [t[i + 1] - t[i] for i in range(n - 1)]
        names = ["in"] + ["qkv", "att", "out", "gin", "gout"] * 6 + ["head"]
        agg = {}
        for i, nm in enumerate(names):
            agg.setdefault(nm, [0, 0, 0])
            agg[nm][0] += 1; agg[nm][1] += d[2 * i]; agg[nm][2] += d[2 * i + 1]
        r["trace_clk_per_phase"] = {k: {"n": v[0], "work_clk": v[1] / v[0], "barrier_clk": v[2] / v[0]} for k, v in agg.items()}
        r["trace_total_clk"] = t[n - 1] - t[0]
        seq = torch.randint(0, 2048, (B, 9, 1), device=dev)
        m.use_cuda_graphs = True
        r["temporal_graph_ms"] = timeit(lambda: (st._advance_host(0), st._replay(("temporal",), st._temporal)), 10)
        r["frame_graph_ms"] = timeit(lambda: m.forward_step(seq), 10)
        st.offset.fill_(2100); st.pos_host[:] = 2100
        m.check_device_errors()
        res[f"B{B}"] = r
        print(B, json.dumps(r), flush=True)
        json.dump(res, open("gpurun_out/r2_depth_timing.json", "w"), indent=1)


for B in (32, 48):
    try:
        one(B)
    except torch.cuda.OutOfMemoryError as e:
        print(B, "OOM")
    m._state = None
    import gc
    gc.collect()
    torch.cuda.empty_cache()
