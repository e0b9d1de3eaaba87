"""Batch TTS over utterances of different lengths (-m gpu): the row-mapped RoPE/KV-append and ring attention kernels, the
per-row sampler, GPT.prefill_streams in a live scope, InferenceImp.generate_many against InferenceImp on each utterance
alone, and `python -m rstnet_b200.offline synthesize`."""
import dataclasses
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import lm_oracle as L
from rstnet_b200 import _lib, ops
from rstnet_b200.lm import GPT, Config

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
BF = torch.bfloat16
TEXT_EMPTY = 128002


@pytest.fixture(scope="module")
def small_lm():
    """L.SMALL (context 16, block_size 64: rings wrap) as in test_lm_gpu.py."""
    cfg = L.SMALL
    w32 = L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05)
    m = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                   intermediate_size=cfg.intermediate_size, norm_eps=cfg.norm_eps, padded_vocab_size=cfg.padded_vocab_size,
                   audio_card=cfg.audio_card, n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim,
                   codecformer_heads=cfg.codecformer_heads, codecformer_layers=cfg.codecformer_layers,
                   codecformer_dim_feedforward=cfg.codecformer_dim_feedforward, context=cfg.context))
    m.load_state_dict(w32, strict=True)
    m.use_cuda_graphs = True
    return m.to(DEV, BF).eval(), {k: v.to(BF) for k, v in w32.items()}, cfg, w32


# ------------------------------------------------------------------------------------------------ 1. row-mapped kernels
@pytest.mark.parametrize("nh,nkv,hs,rope_n", [(4, 4, 64, 64), (8, 2, 128, 96), (6, 2, 64, 32)])
def test_row_mapped_rope_append_and_attention_equal_uniform(nh, nkv, hs, rope_n):
    lib, st = _lib.lib(), ops._stream()
    g = torch.Generator(device="cpu").manual_seed(nh * 100 + hs)
    B, tn, cap, context, rope_rows = 5, 3, 16, 16, 64
    qpk = nh // nkv
    offset = torch.tensor([2, 20, 5, 13, 0], dtype=torch.int64, device=DEV)       # stream 1's ring has wrapped
    qkv_u = torch.randn(tn * B, nkv * (qpk + 2) * hs, generator=g).to(DEV, BF)
    cos = torch.randn(rope_rows, rope_n, generator=g).to(DEV, BF)
    sin = torch.randn(rope_rows, rope_n, generator=g).to(DEV, BF)
    kv0 = torch.randn(2, B, nkv, cap, hs, generator=g).to(DEV, BF)
    # uniform launch over every (tl, stream) pair
    kv_u, q_u, att_u = kv0.clone(), torch.zeros(tn * B, nh * hs, dtype=BF, device=DEV), torch.zeros(tn * B, nh * hs, dtype=BF, device=DEV)
    _lib.check(lib.rstnet_lm_rope_kv_append_bf16(qkv_u.data_ptr(), cos.data_ptr(), sin.data_ptr(), rope_rows, rope_n, offset.data_ptr(), 1,
                                                 None, None, q_u.data_ptr(), kv_u.data_ptr(), tn * B, B, nh, nkv, hs, cap, st))
    _lib.check(lib.rstnet_lm_ring_decode_attention_bf16(q_u.data_ptr(), kv_u.data_ptr(), offset.data_ptr(), 1, None, None, att_u.data_ptr(),
                                                        tn * B, B, nh, nkv, hs, cap, context, st))
    # mapped launch: streams {0, 2, 3} in a shuffled order with padding rows in between; streams 1 and 4 are absent
    pairs = [(b, tl) for b in (0, 2, 3) for tl in range(tn)]
    random.Random(hs).shuffle(pairs)
    rows = pairs[:4] + [(-1, 0)] * 2 + pairs[4:] + [(-1, 0)] * 3
    M = len(rows)
    rs = torch.tensor([b for b, _ in rows], dtype=torch.int32, device=DEV)
    rt = torch.tensor([t for _, t in rows], dtype=torch.int32, device=DEV)
    src = torch.tensor([t * B + b if b >= 0 else 0 for b, t in rows], device=DEV)
    qkv_m = qkv_u[src].contiguous()
    nanb = torch.tensor(float("nan"), dtype=BF)
    kv_m = kv0.clone()
    q_m = torch.full((M, nh * hs), nanb, dtype=BF, device=DEV)
    att_m = torch.full((M, nh * hs), nanb, dtype=BF, device=DEV)
    _lib.check(lib.rstnet_lm_rope_kv_append_bf16(qkv_m.data_ptr(), cos.data_ptr(), sin.data_ptr(), rope_rows, rope_n, offset.data_ptr(), 1,
                                                 rs.data_ptr(), rt.data_ptr(), q_m.data_ptr(), kv_m.data_ptr(), M, B, nh, nkv, hs, cap, st))
    _lib.check(lib.rstnet_lm_ring_decode_attention_bf16(q_m.data_ptr(), kv_m.data_ptr(), offset.data_ptr(), 1, rs.data_ptr(), rt.data_ptr(),
                                                        att_m.data_ptr(), M, B, nh, nkv, hs, cap, context, st))
    torch.cuda.synchronize()
    bits = lambda t: t.view(torch.int16)
    for r, (b, t) in enumerate(rows):
        if b < 0:
            assert torch.isnan(q_m[r].float()).all() and torch.isnan(att_m[r].float()).all(), r     # padding rows: nothing written
        else:
            assert torch.equal(bits(q_m[r]), bits(q_u[t * B + b])), (r, b, t)
            assert torch.equal(bits(att_m[r]), bits(att_u[t * B + b])), (r, b, t)
    for b in (0, 2, 3):
        assert torch.equal(bits(kv_m[:, b]), bits(kv_u[:, b])), b
    for b in (1, 4):
        assert torch.equal(bits(kv_m[:, b]), bits(kv0[:, b])), b
    assert torch.equal(offset.cpu(), torch.tensor([2, 20, 5, 13, 0]))


def test_counter_add_rows():
    c = torch.arange(300, dtype=torch.int64, device=DEV)
    d = torch.randint(0, 50, (300,), dtype=torch.int64, device=DEV)
    ref = c + d
    _lib.check(_lib.lib().rstnet_counter_add_rows(c.data_ptr(), d.data_ptr(), 300, ops._stream()))
    assert torch.equal(c, ref)


# ------------------------------------------------------------------------------------------------ 3. per-row sampler
def _sample(logits, rows, V, n_valid, top_k, temp, seed, out, counter=None, nv_table=None, nv_stride=0, steps=None, keys=None):
    """rstnet_lm_sample_params_bf16 without settings tables or top_p: the RNG keyed by (seed, *counter, row), or by
    (seed, steps[row], keys[row]) when those are given; candidates n_valid, or nv_table[row * nv_stride] when given"""
    p = lambda t: None if t is None else t.data_ptr()
    _lib.check(_lib.lib().rstnet_lm_sample_params_bf16(logits.data_ptr(), rows, V, n_valid, p(nv_table), nv_stride, top_k, temp, 0.0,
                                                       None, None, None, 0, seed, p(counter), p(steps), p(keys), out.data_ptr(), 1,
                                                       ops._stream()))


@pytest.mark.parametrize("V", [2050, 20000])
def test_row_sampler_equals_uniform_sampler(V):
    """the sampler's per-row RNG and per-row candidate-count forms equal its scalar form"""
    rows, seed, step = 37, 77, 9
    g = torch.Generator(device="cpu").manual_seed(V)
    logits = (torch.randn(rows, V, generator=g) * 2).to(DEV, BF)
    logits[3, :] = 0.5                                                       # an all-tie row
    keys = torch.arange(rows, dtype=torch.int32, device=DEV)
    steps = torch.full((rows,), step, dtype=torch.int64, device=DEV)
    counter = torch.tensor([step], dtype=torch.int64, device=DEV)

    def uniform(n_valid, top_k, temp):
        out = torch.full((rows,), -1, dtype=torch.int64, device=DEV)
        _sample(logits, rows, V, n_valid, top_k, temp, seed, out, counter=counter)
        return out

    def per_row(nv_table, n_valid, top_k, temp):
        out = torch.full((rows,), -1, dtype=torch.int64, device=DEV)
        _sample(logits, rows, V, n_valid, top_k, temp, seed, out, nv_table=nv_table, nv_stride=2, steps=steps, keys=keys)
        return out

    for top_k, temp in ((0, 1.0), (1, 0.8), (30, 0.8), (64, 1.3), (100, 0.8), (1024, 0.7), (-1, 0.9)):
        for n_valid in (2048, V):
            ref = uniform(n_valid, top_k, temp)
            assert torch.equal(per_row(None, n_valid, top_k, temp), ref), (top_k, n_valid)
            table = torch.full((rows, 2), 1, dtype=torch.int32, device=DEV)     # column 0 read (stride 2)
            table[:, 0] = n_valid
            assert torch.equal(per_row(table, V, top_k, temp), ref), (top_k, n_valid)
        # mixed per-row candidate counts: each row equals the uniform sampler at its own n_valid
        choices = [2048, 2049, 1500, 40, V, 0]          # 0: the whole row, as the uniform form reads n_valid <= 0
        nv = torch.tensor([choices[r % len(choices)] for r in range(rows)], dtype=torch.int32)
        table = torch.stack([nv, torch.ones_like(nv)], 1).to(DEV)
        got = per_row(table, V, top_k, temp)
        for c in choices:
            ref = uniform(c, top_k, temp)
            sel = (nv == c).nonzero().flatten().to(DEV)
            assert torch.equal(got[sel], ref[sel]), (top_k, c)
    # keys and steps select the random stream: a row keyed k at step s draws what uniform row k draws at counter s
    perm = torch.randperm(rows, generator=g)
    keys2 = perm.to(torch.int32).to(DEV)
    lg2 = logits[perm.to(DEV)].contiguous()
    out = torch.full((rows,), -1, dtype=torch.int64, device=DEV)
    _sample(lg2, rows, V, V, 30, 0.8, seed, out, steps=steps, keys=keys2)
    assert torch.equal(out, uniform(V, 30, 0.8)[perm.to(DEV)])


# ------------------------------------------------------------------------------------------------ 2. prefill_streams
def _snapshot(st):
    return [k.clone() for k in st.kv], st.offset.clone(), st.pos_host.copy(), st.active.clone(), st.active_host.copy()


def _restore(st, snap):
    for k, s in zip(st.kv, snap[0]):
        k.copy_(s)
    st.offset.copy_(snap[1])
    st.pos_host[:] = snap[2]
    st.active.copy_(snap[3])
    st.active_host[:] = snap[4]


def test_prefill_streams_in_live_scope(small_lm):
    m, w, cfg, _ = small_lm
    B, cap = 6, cfg.context
    g = torch.Generator().manual_seed(21)
    prompts = {1: torch.randint(0, 2048, (9, 5), generator=g), 4: torch.randint(0, 2048, (9, 20), generator=g)}   # 20 > ring
    for p in prompts.values():
        p[0] = torch.randint(0, 1000, (p.shape[1],), generator=g)
    nxt = torch.randint(0, 2048, (B, 9, 1), generator=g).to(DEV)
    with m.streaming(B):
        st = m._state
        for f in range(22):        # every stream mid-run at its own position; streams 0, 2, 5 wrap their rings
            m.set_active_streams([1, f % 2, 1, int(f % 3 == 0), int(f < 9), 1])
            m.forward_step(torch.randint(0, 2048, (B, 9, 1), generator=g).to(DEV), use_sampling=False)
        m.set_active_streams([1, 0, 1, 1, 0, 1])
        pos0 = st.pos_host.copy()
        assert pos0.max() > cap
        snap = _snapshot(st)
        m.reset_streaming(streams=[1, 4])
        m.prefill_streams({s: p.to(DEV) for s, p in prompts.items()})
        torch.cuda.synchronize()
        others = [0, 2, 3, 5]
        for l in range(cfg.n_layer):
            assert torch.equal(st.kv[l][:, others], snap[0][l][:, others])
        off = st.offset.cpu().numpy()
        assert list(off[others]) == list(pos0[others]) and off[1] == 5 and off[4] == 20
        assert list(st.pos_host) == list(off)
        assert torch.equal(st.active, snap[3]) and list(st.active_host) == list(snap[4])
        rings = {s: [k[:, s].clone() for k in st.kv] for s in prompts}
        t_after = m.forward_step(nxt, use_sampling=False)
        _restore(st, snap)
        t_before = m.forward_step(nxt, use_sampling=False)
        assert torch.equal(t_after[others], t_before[others])
    # the prefilled streams' rings == the same prompts fed one position at a time in a fresh scope
    for s, p in prompts.items():
        T = p.shape[1]
        with m.streaming(1):
            for t in range(T):
                m.forward_global(p[None, :, t:t + 1].to(DEV))
            fresh = [k[:, 0] for k in m._state.kv]
            slots = list(range(min(T, cap)))
            for l in range(cfg.n_layer):
                assert torch.equal(rings[s][l][:, :, slots], fresh[l][:, :, slots]), (s, l)


# ------------------------------------------------------------------------------------------------ 4./5. generate_many
def _corpus(n, seed, pmax=20, gmax=12):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        P = int(torch.randint(3, pmax + 1, (1,), generator=g))
        G = int(torch.randint(2, gmax + 1, (1,), generator=g))
        seq = torch.randint(0, 2048, (9, P + G), generator=g)
        seq[0, :P] = torch.randint(0, 1000, (P,), generator=g)
        seq[0, P:] = TEXT_EMPTY
        if i % 3 == 0:                                          # trailing pad frames are stripped
            seq = torch.cat([seq, torch.full((9, 2), 2049)], 1)
        out.append((f"utt{i}", seq))
    return out


def _imp(m, use_sampling, tk_text=25, tk=30):
    from rstnet_b200.infer import InferenceImp
    imp = InferenceImp(None, m, "sampling", 0.7, tk_text, 0.8, tk, "TTS")
    imp.use_sampling = use_sampling
    return imp


@pytest.mark.parametrize("mode,use_sampling,tk", [("greedy", False, 0), ("top1", True, 1), ("sampled", True, 30)])
def test_generate_many_equals_each_utterance_alone(golden_dir, small_lm, mode, use_sampling, tk):
    from test_lm_gpu import _replay_ok
    m, w, cfg, _ = small_lm
    gold = np.load(os.path.join(golden_dir, "lm_round2.npz"))
    corpus = _corpus(12, 5) + [("golden", torch.from_numpy(gold["infer_seq"]))]
    imp = _imp(m, use_sampling, tk, tk) if tk <= 1 else _imp(m, True)
    alone = {}
    for utt, seq in corpus:
        codes, raw = imp.generate(seq.unsqueeze(0).to(DEV), return_frames=True)
        alone[utt] = (codes[0].cpu(), raw[0].cpu())
    for cap in (1, 4, 7, 20):
        got = list(imp.generate_many(((u, s.to(DEV)) for u, s in corpus), cap, return_frames=True))
        assert sorted(u for u, _, _ in got) == sorted(u for u, _ in corpus)
        for utt, codes, raw in got:
            assert torch.equal(codes.cpu(), alone[utt][0]), (cap, utt)
            assert torch.equal(raw.cpu(), alone[utt][1]), (cap, utt)
    if mode == "sampled":
        return      # the oracle restates the deterministic decisions only (argmax / top-1)
    # the golden utterance: the reference's own bf16 tokens up to the first near-tie (test_inference_imp_vs_reference_loop)
    tol = 0.07
    margins = torch.from_numpy(gold[f"infer_bf16_{mode}_margins"]).flatten()
    ref = torch.from_numpy(gold[f"infer_bf16_{mode}_frames"]).flatten()
    first_tie = int((margins <= tol).nonzero()[0]) if bool((margins <= tol).any()) else margins.numel()
    assert torch.equal(alone["golden"][1].flatten()[:first_tie], ref[:first_tie])
    exact, n = _replay_ok(alone["golden"][1], torch.from_numpy(gold["infer_seq"]), w, cfg, use_sampling, tol)
    assert exact >= 0.8 * n
    # every decision of two short utterances (P + G < 16) under the oracle replay
    short = [(u, s) for u, s in corpus[:12] if s.shape[1] < 16][:2]
    assert len(short) == 2
    for utt, seq in short:
        exact, n = _replay_ok(alone[utt][1], seq, w, cfg, use_sampling, tol)
        assert exact >= 0.8 * n


def test_generate_many_capacity_above_128(small_lm):
    """130 rows: the decode steps run the 256-column GEMM; checked decision by decision under the oracle."""
    from test_lm_gpu import _replay_ok
    m, w, cfg, _ = small_lm
    corpus = _corpus(150, 9, pmax=8, gmax=5)
    imp = _imp(m, False)
    got = {u: (c, r) for u, c, r in imp.generate_many(((u, s.to(DEV)) for u, s in corpus), 130, return_frames=True)}
    assert sorted(got) == sorted(u for u, _ in corpus)
    seqs = dict(corpus)
    exact = n = 0
    for utt in [f"utt{i}" for i in range(0, 150, 10)] + ["utt129", "utt149"]:
        seq = seqs[utt]
        e, k = _replay_ok(got[utt][1].cpu(), seq, w, cfg, False, 0.07)
        exact, n = exact + e, n + k
    assert exact >= 0.8 * n


# ------------------------------------------------------------------------------------------------ 6. CLI
def test_synthesize_cli_equals_generate_many(small_lm, tmp_path):
    from rstnet_b200 import offline
    m, w, cfg, w32 = small_lm
    (tmp_path / "gpt.json").write_text(json.dumps(dataclasses.asdict(m.config)))
    torch.save({"model": {"module." + k: v for k, v in w32.items()}}, tmp_path / "ckpt.pt")
    corpus = dict(_corpus(6, 13))
    torch.save(corpus, tmp_path / "corpus.pt")
    assert offline.main(["synthesize", "--input", str(tmp_path / "corpus.pt"), "--config", str(tmp_path / "gpt.json"),
                         "--checkpoint", str(tmp_path / "ckpt.pt"), "--output-file", str(tmp_path / "codes.pt"),
                         "--capacity", "4", "--device", "cuda:0"]) == 0
    got = torch.load(tmp_path / "codes.pt")
    ref = dict(_imp(m, True).generate_many(((u, s.to(DEV)) for u, s in corpus.items()), 4))
    assert sorted(got) == sorted(corpus)
    for u, c in got.items():
        assert c.dtype == torch.int16 and c.dim() == 2 and c.shape[0] == 8
        assert torch.equal(c.to(torch.int64), ref[u].cpu()), u
