"""CPU tests of prompted Moshi generation: `moshi.prompt_from_aligned` against a hand-written loop, a host restatement of
the delay-cache prompt kernel's contract (LMGen.step's cache rule run P times) against the closed form of what the
temporal transformer is fed, the new C entry points' declarations, bindings and argument errors, and the argument errors
of `LMGen.prefill_streams`, `generate_many`, `FrameScheduler.admit(prompt=)` and `offline continue`."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from rstnet_b200 import _lib
from rstnet_b200._lib import RstnetError
from rstnet_b200.moshi import LMGen, LMModel, _item, generate_many, prompt_from_aligned

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DELAYS = {0: (0,) * 7, 1: (0, 0, 1, 1, 0, 1, 1), 2: (0, 1, 2, 0, 0, 2, 1)}   # K = 7, dep_q = 3, by max_delay
DEP_Q = 3
TEXT_INIT, AUDIO_INIT = 500, 64


def _aligned(K, L, seed):
    return torch.randint(0, 60, (K, L), generator=torch.Generator().manual_seed(seed))


def _hand_prompt(seq, P, delays, dep_q, initial=-2):
    K = seq.shape[0]
    out = [[initial] * P for _ in range(K)]
    for k in range(K):
        for t in range(P):
            if k > dep_q:
                out[k][t] = int(seq[k, t])
            elif t >= delays[k]:
                out[k][t] = int(seq[k, t - delays[k]])
    return torch.tensor(out, dtype=torch.int64).reshape(K, P)


@pytest.mark.parametrize("md", [0, 1, 2])
@pytest.mark.parametrize("P", [0, 1, 2, 3, 9])
def test_prompt_from_aligned_vs_hand_loop(md, P):
    delays = DELAYS[md]
    seq = _aligned(len(delays), 12, 10 * md + P)
    got = prompt_from_aligned(seq, P, delays, DEP_Q)
    assert got.dtype == torch.int64 and got.shape == (len(delays), P)
    assert torch.equal(got, _hand_prompt(seq, P, delays, DEP_Q))
    assert torch.equal(prompt_from_aligned(seq, P, delays, DEP_Q, initial=77), _hand_prompt(seq, P, delays, DEP_Q, 77))


def test_prompt_from_aligned_rejects_bad_arguments():
    seq = _aligned(7, 5, 0)
    for bad in [dict(P=6), dict(P=-1), dict(delays=(0,) * 6), dict(dep_q=7), dict(seq=seq.float()), dict(seq=seq[0])]:
        kw = dict(seq=seq, P=2, delays=DELAYS[1], dep_q=DEP_Q)
        kw.update(bad)
        with pytest.raises(RstnetError):
            prompt_from_aligned(kw["seq"], kw["P"], kw["delays"], kw["dep_q"])


# ------------------------------------------------------------------------------- the prompt kernel's contract, on the host
def restate_prompt(cache, off, delays, prompt, dep_q, text_init, audio_init):
    """One row: P steps of cache_in then cache_out (csrc/delay_cache.cu) from (cache [K, CT], off), with the user tokens
    and the sampled tokens taken from prompt [K, P].  -> (feed [P, K], cache, off, valid)."""
    cache = cache.clone()
    K, CT = cache.shape
    P = prompt.shape[1]
    max_delay = CT - 2
    feed = torch.empty(P, K, dtype=torch.int64)
    o = int(off)
    for t in range(P):
        for k in range(dep_q + 1, K):
            cache[k, (o + delays[k]) % CT] = prompt[k, t]
        for k in range(K):
            if o <= delays[k]:
                cache[k, o % CT] = text_init if k == 0 else audio_init
        feed[t] = cache[:, o % CT]
        o += 1
        cache[:dep_q + 1, o % CT] = prompt[:dep_q + 1, t]
    return feed, cache, o, int(o > max_delay)


@pytest.mark.parametrize("md", [0, 1, 2])
@pytest.mark.parametrize("P", [1, 2, 3, 11])
def test_prompt_restatement_feeds_the_aligned_inputs(md, P):
    """From a reset row, the feed at step t is the aligned frame the model conditions on: codebook k <= dep_q the frame
    t - 1 - d_k of Moshi's channels, a user codebook the frame t - d_k, the initial token while t <= d_k; the final
    cache holds the prompt's last columns, off = P, valid = P > max_delay."""
    delays = DELAYS[md]
    K, CT = len(delays), md + 2
    seq = _aligned(K, P + 4, 100 + P)
    prompt = prompt_from_aligned(seq, P, delays, DEP_Q)
    cache0 = torch.full((K, CT), -2, dtype=torch.int64)
    feed, cache, off, valid = restate_prompt(cache0, 0, delays, prompt, DEP_Q, TEXT_INIT, AUDIO_INIT)
    for t in range(P):
        for k in range(K):
            d = delays[k]
            if t <= d:
                want = TEXT_INIT if k == 0 else AUDIO_INIT
            else:
                want = seq[k, t - 1 - d] if k <= DEP_Q else seq[k, t - d]
            assert int(feed[t, k]) == int(want), (t, k)
    assert off == P and valid == int(P > md)
    for k in range(DEP_Q + 1):       # the last step's sampled tokens are in column P
        assert int(cache[k, P % CT]) == int(prompt[k, P - 1])


def test_prompt_restatement_composes():
    """Two prompts back to back equal one prompt of their concatenation (the contract starts from any state)."""
    delays = DELAYS[2]
    K, CT = len(delays), 4
    prompt = prompt_from_aligned(_aligned(K, 20, 7), 20, delays, DEP_Q)
    c0 = torch.randint(-2, 60, (K, CT), generator=torch.Generator().manual_seed(3))
    f, c, o, v = restate_prompt(c0, 1, delays, prompt, DEP_Q, TEXT_INIT, AUDIO_INIT)
    f1, c1, o1, _ = restate_prompt(c0, 1, delays, prompt[:, :7], DEP_Q, TEXT_INIT, AUDIO_INIT)
    f2, c2, o2, v2 = restate_prompt(c1, o1, delays, prompt[:, 7:], DEP_Q, TEXT_INIT, AUDIO_INIT)
    assert torch.equal(torch.cat([f1, f2]), f) and torch.equal(c2, c) and (o2, v2) == (o, v) == (21, 1)


# ------------------------------------------------------------------------------- the C ABI
def test_abi_declares_binds_and_exports_the_new_entry_points():
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    for name, n in (("rstnet_lm_delay_cache_prompt", 20), ("rstnet_lm_rope_pair_kv_append_paged_rows_bf16", 16)):
        assert f"int {name}(" in header and name in _lib.SYMBOLS
        assert len(getattr(_lib.lib(), name).argtypes) == n
    assert "#define RSTNET_DELAY_PROMPT_MAX_ROWS 256" in header and _lib.DELAY_PROMPT_MAX_ROWS == 256
    integration = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert "rstnet_lm_delay_cache_prompt" in integration and "rstnet_lm_rope_pair_kv_append_paged_rows_bf16" in integration


def _arr(*v):
    return np.array(v, dtype=np.int32)


def _prompt_call(**kw):
    """rstnet_lm_delay_cache_prompt with fake (never dereferenced) device pointers: every case below is refused before
    any launch"""
    a = dict(cache=8, off=8, valid=8, delays=8, prompt=8, prompt_stride=7, feed=8, feed_stride=7, rows=_arr(0, 1),
             starts=_arr(0, 3), lengths=_arr(3, 2), n=2, B=4, K=7, dep_q=3, CT=4, max_delay=2)
    a.update(kw)
    ptr = lambda x: x.ctypes.data if isinstance(x, np.ndarray) else x
    return _lib.lib().rstnet_lm_delay_cache_prompt(
        a["cache"], a["off"], a["valid"], a["delays"], a["prompt"], a["prompt_stride"], a["feed"], a["feed_stride"],
        ptr(a["rows"]), ptr(a["starts"]), ptr(a["lengths"]), a["n"], a["B"], a["K"], a["dep_q"], a["CT"], a["max_delay"],
        TEXT_INIT, AUDIO_INIT, None)


@pytest.mark.parametrize("bad,msg", [
    (dict(cache=None), b"null pointer"), (dict(feed=None), b"null pointer"), (dict(rows=None), b"null pointer"),
    (dict(n=-1), b"rows"), (dict(n=257), b"rows"), (dict(CT=3), b"bad shape"), (dict(K=129), b"bad shape"),
    (dict(dep_q=7), b"bad shape"), (dict(prompt_stride=6), b"strides"), (dict(feed_stride=6), b"strides"),
    (dict(rows=_arr(0, 4)), b"outside"), (dict(rows=_arr(-1, 0)), b"outside"), (dict(rows=_arr(2, 2)), b"twice"),
    (dict(lengths=_arr(3, -1)), b"negative"), (dict(starts=_arr(-3, 0)), b"negative"),
])
def test_delay_cache_prompt_refuses_bad_arguments(bad, msg):
    assert _prompt_call(**bad) != 0
    assert msg in _lib.lib().rstnet_last_error()


def test_delay_cache_prompt_with_only_empty_prompts_launches_nothing():
    before = _lib.launch_count()
    assert _prompt_call(lengths=_arr(0, 0)) == 0 and _prompt_call(n=0) == 0
    assert _lib.launch_count() == before


def test_paged_rows_rope_refuses_bad_arguments():
    L = _lib.lib()
    args = lambda **kw: [kw.get(n, d) for n, d in (("qkv", 8), ("offset", 8), ("rs", 8), ("rt", 8), ("q", 8), ("kv", 8),
                                                   ("rows", 16), ("B", 4), ("H", 4), ("hd", 64), ("cap", 16), ("freqs", 8),
                                                   ("table", 8), ("stride", 1), ("log2", 4))] + [None]
    for bad, msg in [(dict(rs=None), b"row map"), (dict(rt=None), b"row map"), (dict(table=None), b"page table"),
                     (dict(log2=3), b"log2_page"), (dict(cap=17), b"do not cover"), (dict(qkv=None), b"null pointer"),
                     (dict(rows=0), b"bad shape"), (dict(hd=63), b"bad shape")]:
        assert L.rstnet_lm_rope_pair_kv_append_paged_rows_bf16(*args(**bad)) != 0, bad
        assert msg in L.rstnet_last_error(), (bad, L.rstnet_last_error())


# ------------------------------------------------------------------------------- Python argument errors
def _small_lm():
    return LMModel(delays=list(DELAYS[1]), n_q=6, dep_q=DEP_Q, card=60, text_card=500, dim=64, num_heads=2, num_layers=1,
                   hidden_scale=4.125, norm="rms_norm_f32", gating="silu", positional_embedding="rope", depformer_dim=64,
                   depformer_dim_feedforward=128, depformer_num_heads=2, depformer_num_layers=1, depformer_multi_linear=True,
                   depformer_weights_per_step=True, depformer_pos_emb="none", existing_text_padding_id=3, context=16)


def test_lmgen_prefill_streams_argument_errors():
    gen = LMGen(_small_lm(), use_sampling=False)
    with pytest.raises(ValueError):
        gen.prefill_streams({0: torch.zeros(7, 2, dtype=torch.int64)})          # not streaming
    # a stand-in scope of 4 rows with a paged allocator whose rows hold 3 positions: every check runs before any launch
    pages = SimpleNamespace(check=lambda s, p, n: (_ for _ in ()).throw(RstnetError("holds KV pages")) if n > 3 else None)
    gen._st = SimpleNamespace(B=4, lm=SimpleNamespace(pages=pages, pos_host=np.zeros(4, dtype=np.int64)))
    z = lambda *s: torch.zeros(*s, dtype=torch.int64)
    for bad in [{4: z(7, 2)}, {-1: z(7, 2)}, {0: z(6, 2)}, {0: z(7)}, {0: z(7, 2).float()}, {0: z(7, 2).bool()},
                {0: np.zeros((7, 2))}, {1: z(7, 4)}]:
        with pytest.raises(RstnetError):
            gen.prefill_streams(bad)
    assert gen._prompt_begin({0: z(7, 0), 1: z(7, 0)}) == []                  # P = 0: nothing to do, nothing launched


def test_generate_many_argument_errors():
    lm = _small_lm()
    gen = LMGen(lm, use_sampling=False)
    for kw in [dict(capacity=0), dict(capacity=257), dict(capacity=2.0), dict(capacity=True), dict(capacity=2, seeds=[1]),
               dict(capacity=2, sampling={"a": 1})]:
        cap = kw.pop("capacity")
        with pytest.raises(RstnetError):
            next(generate_many(gen, [], cap, **kw))
    gen._st = object()
    with pytest.raises(RstnetError, match="not streaming"):
        next(generate_many(gen, [], 2))
    seq = torch.zeros(7, 5, dtype=torch.int64)
    assert _item(("u", seq, 4), 7)[2] == 4
    for bad in [("u", seq, 5), ("u", seq, -1), ("u", seq, 1.0), ("u", seq, True), ("u", seq[:6], 1), ("u", seq.float(), 1),
                ("u", seq), None]:
        with pytest.raises(RstnetError):
            _item(bad, 7)


class _FakeEngine:
    """the engine half FrameScheduler drives, recording restarts"""

    def __init__(self, free_pages=None, moshi=True):
        self.kv_pages = None if free_pages is None else 100
        self.kv_pages_free = free_pages
        self.calls = []
        self.prefilling = frozenset()
        if moshi:
            self.check_prompt = lambda p: int(p.shape[1]) if torch.is_tensor(p) and p.dim() == 2 and p.shape[0] == 7 else \
                (_ for _ in ()).throw(RstnetError("a prompt is an integer tensor [7, P]"))

    def kv_pages_for(self, positions):
        return -(-positions // 16)

    def reset_rows(self, *a, **kw):
        self.calls.append(("reset", a, kw))

    def start_rows(self, *a, **kw):
        self.calls.append(("start", a, kw))


def test_scheduler_admit_with_prompt_argument_errors_change_nothing():
    from rstnet_b200.serve import FrameScheduler
    p = torch.zeros(7, 40, dtype=torch.int64)
    for eng, prompt, exc in [(_FakeEngine(moshi=False), p, RstnetError), (_FakeEngine(), p[:6], RstnetError),
                             (_FakeEngine(free_pages=3), p, RuntimeError),                  # needs 3 + headroom 1
                             (_FakeEngine(free_pages=3), p[:, :47], RuntimeError)]:
        fs = FrameScheduler(eng, 4, kv_headroom=1)
        with pytest.raises(exc):
            fs.admit("s", prompt=prompt)
        assert eng.calls == [] and fs.free_rows() == 4 and fs.sessions() == {}
    eng = _FakeEngine(free_pages=4)
    fs = FrameScheduler(eng, 4, kv_headroom=1)
    assert fs.admit("s", seed=3, prompt=p) == 0
    assert eng.calls[0][0] == "start" and eng.calls[0][2]["prompts"][0] is p and eng.calls[0][2]["seed"] == 3


def test_gpt_duplex_engine_refuses_prompts():
    from rstnet_b200.serve import DuplexEngine
    eng = DuplexEngine.__new__(DuplexEngine)
    with pytest.raises(RstnetError, match="MoshiDuplexEngine"):
        eng.reset_rows([0], prompts={0: torch.zeros(9, 2, dtype=torch.int64)})


def test_continue_cli_parser():
    from rstnet_b200.offline import build_parser
    base = ["continue", "--model", "moshi", "--config", "c.json", "--checkpoint", "ck", "--input", "in.pt", "--output-file", "o.pt"]
    a = build_parser().parse_args(base + ["--prompt-frames", "25", "--capacity", "8", "--kv-gb", "2", "--seed", "4"])
    assert (a.cmd, a.prompt_frames, a.capacity, a.kv_gb, a.seed, a.wav_dir) == ("continue", 25, 8, 2.0, 4, None)
    for bad in [base, base + ["--prompt-frames", "-1"], base + ["--prompt-frames", "x"], base + ["--prompt-frames", "2", "--kv-gb", "0"],
                [b if b != "moshi" else "gpt" for b in base] + ["--prompt-frames", "2"]]:
        with pytest.raises(SystemExit):
            build_parser().parse_args(bad)
