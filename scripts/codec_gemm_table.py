"""Per-shape table of the codec's tensor-core GEMM launches over one streaming frame (256 streams): time, FLOP/s, bytes/s."""
import sys, json
import torch
sys.path.insert(0, ".")
import bench
from rstnet_b200 import ops

dev = torch.device("cuda", 0)
B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
from specs import mimi_spec as S
m = bench._mimi(dev, S)
rec = []
orig_init, orig_run = ops.TcGemm.__init__, ops.TcGemm.run


def init(self, A, a_off, a_i_stride, a_o_stride, a_c_extent, a_i_extent, a_o_extent, W, Kc, C_, c_off, c_i_stride, c_o_stride, I_out, O_out, **kw):
    orig_init(self, A, a_off, a_i_stride, a_o_stride, a_c_extent, a_i_extent, a_o_extent, W, Kc, C_, c_off, c_i_stride, c_o_stride, I_out, O_out, **kw)
    self.shape = dict(M=I_out * O_out, I=I_out, O=O_out, N=W.shape[0], K=W.shape[1], taps=kw.get("taps", 1), o_mul=kw.get("o_mul", 1),
                      nsplit=kw.get("n_split", 0), pre=kw.get("pre_act", 0), post=kw.get("post_act", 0), R=kw.get("R") is not None,
                      C2=kw.get("C2") is not None, prec=kw.get("precision", 0))


def run(self):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); orig_run(self); e1.record()
    rec.append((e0, e1, self))


ops.TcGemm.__init__ = init
ops.TcGemm.run = run
m.use_cuda_graphs = False
m.streaming_forever(B)
x = torch.randn(B, 1, 1920 * 4, device=dev)
with torch.no_grad():
    for i in range(2):
        c = m.encode(x[..., i * 1920:(i + 1) * 1920]); m.decode(c)
    torch.cuda.synchronize(); rec.clear()
    n = 3
    for i in range(n):
        torch.cuda._sleep(20_000_000)
        c = m.encode(x[..., (i + 1) * 1920:(i + 2) * 1920]); m.decode(c)
    torch.cuda.synchronize()
rows = {}
for e0, e1, p in rec:
    key = json.dumps(p.shape)
    d = rows.setdefault(key, [0, 0.0, p])
    d[0] += 1; d[1] += e0.elapsed_time(e1)
tot = sum(v[1] for v in rows.values()) / n
print(f"total GEMM time per frame {tot*1e3:.0f} us over {len(rec)//n} launches")
print(f"{'us/launch':>9} {'n':>3} {'%':>5} {'TF/s':>6} {'TB/s':>5}  shape")
for key, (cnt, ms, p) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
    us = ms * 1e3 / cnt
    print(f"{us:9.1f} {cnt//n:3d} {100*ms/n/tot:5.1f} {p.flops/us/1e6:6.1f} {p.bytes/us/1e6:5.2f}  {key}")
