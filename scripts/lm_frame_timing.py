"""Time one LM frame (7B shapes, B = 32, full 2048-key ring): temporal graph and whole-frame graph."""
import json
import os
import sys

import torch

sys.path.insert(0, ".")
import bench

dev = torch.device("cuda", 0)
m = bench._gpt7b(dev, context=2048)
B = int(os.environ.get("LM_B", "32"))


def timeit(fn, n=20):
    for _ in range(4):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


with m.streaming(B):
    st = m._state
    for kv in st.kv:
        kv.normal_()
    st.offset.fill_(2100); st.pos_host[:] = 2100
    seq = torch.randint(0, 2048, (B, 9, 1), device=dev)
    r = {"B": B}
    r["temporal_graph_ms"] = timeit(lambda: (st._replay(("temporal",), st._temporal)))
    st.offset.fill_(2100)
    r["frame_graph_ms"] = timeit(lambda: m.forward_step(seq))
    st.offset.fill_(2100); st.pos_host[:] = 2100
    toks = m.forward_step(seq, use_sampling=False)
    r["tok_checksum"] = int(toks.sum())
    m.check_device_errors()
    print(json.dumps(r))
