"""Cost of the sampler's modes on the H100: per-launch time of rstnet_lm_sample_params_bf16 (argmax, top-k 25, top-k 250,
top-p 0.9, multinomial) on text rows (V = 152 064) and audio rows (V = 2 050, 8 heads per stream) at 32 / 128 / 256
streams, and the B = 32 7B-shape frame graph (as scripts/lm_frame_timing.py) with top-k against top-p settings,
alternated in one run.  Prints the card and its power limit with the numbers (one JSON line).

    python scripts/sampling_bench.py [--launches 200] [--frames 30] [--rounds 5]
"""
import argparse
import json
import subprocess
import sys

import torch

sys.path.insert(0, ".")

from rstnet_b200 import _lib, ops  # noqa: E402

DEV = torch.device("cuda", 0)
MODES = {"argmax": (0, 1.0, 0.0), "topk25": (25, 0.8, 0.0), "topk250": (250, 0.8, 0.0), "topp0.9": (-1, 0.8, 0.9),
         "multinomial": (-1, 0.8, 0.0)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def launch_us(logits, mode, n):
    R, V = logits.shape
    tk, temp, tp = mode
    out = torch.zeros(R, dtype=torch.int64, device=DEV)
    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    L = _lib.lib()

    def go():
        _lib.check(L.rstnet_lm_sample_params_bf16(logits.data_ptr(), R, V, 0, None, 1, tk, temp, tp, None, None, None, 1, 1,
                                                  step.data_ptr(), None, None, out.data_ptr(), 1, ops._stream()))
    for _ in range(5):
        go()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        go()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--frames", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    res = {"card": card(), "sampler_us": {}}
    g = torch.Generator(device="cpu").manual_seed(0)
    for B in (32, 128, 256):
        # LM-head-like rows: a Gumbel spread (heavy upper tail) so the nucleus at 0.9 holds a few hundred to thousands of ids
        text = (-torch.empty(B, 152064).exponential_(generator=g).log()).mul(1.5).to(torch.bfloat16).to(DEV)
        audio = (-torch.empty(8 * B, 2050).exponential_(generator=g).log()).mul(1.5).to(torch.bfloat16).to(DEV)
        for name, mode in MODES.items():
            res["sampler_us"][f"text_B{B}_{name}"] = round(launch_us(text, mode, a.launches), 2)
            res["sampler_us"][f"audio_B{B}x8_{name}"] = round(launch_us(audio, mode, a.launches), 2)
    del text, audio
    import bench
    m = bench._gpt7b(DEV, context=2048)
    B = 32
    frames = {"topk": dict(top_k_text=25, top_k=250), "topp": dict(top_k_text=25, top_k=250, top_p_text=0.9, top_p=0.9)}
    times = {k: [] for k in frames}
    with m.streaming(B):
        st = m._state
        for kv in st.kv:
            kv.normal_()
        seq = torch.randint(0, 2048, (B, 9, 1), device=DEV)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for r in range(a.rounds):
            for name, kw in frames.items():
                st.offset.fill_(2100)
                st.pos_host[:] = 2100
                for _ in range(3):
                    m.forward_step(seq, **kw)
                st.offset.fill_(2100)
                st.pos_host[:] = 2100
                torch.cuda.synchronize()
                e0.record()
                for _ in range(a.frames):
                    m.forward_step(seq, **kw)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / a.frames)
        m.check_device_errors()
    res["frame_B32_ms"] = {k: {"min": round(min(v), 4), "median": round(sorted(v)[len(v) // 2], 4)} for k, v in times.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
