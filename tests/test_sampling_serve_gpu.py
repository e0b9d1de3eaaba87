"""Per-session sampling settings in the serving layer (-m gpu): `DuplexEngine` and `MoshiDuplexEngine` driven through
`FrameScheduler.admit(session, sampling=, seed=)`.  A session with its own settings and seed gets the same tokens and PCM
whichever row it is leased and whichever tick it is admitted, beside sessions with other settings and sessions with
none; a session admitted without settings after the switch samples with the engine's defaults and key 0."""
import pytest
import torch

from rstnet_b200.lm import Sampling

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
F = 1920
TICKS = 7


@pytest.fixture(scope="module")
def codec(official_weights):
    from rstnet_b200.codec import MimiCodec
    c = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    c.load_state_dict(official_weights, strict=True)
    c = c.to(DEV).eval()
    c.use_cuda_graphs, c.streaming_tensor_cores = True, True
    yield c
    c._stream_state = None


@pytest.fixture(scope="module")
def gpt():
    from oracle import lm_oracle as L
    from rstnet_b200.lm import GPT, Config
    cfg = L.SMALL
    m = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                   intermediate_size=cfg.intermediate_size, padded_vocab_size=cfg.padded_vocab_size, audio_card=cfg.audio_card,
                   n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim, codecformer_heads=cfg.codecformer_heads,
                   codecformer_layers=cfg.codecformer_layers, codecformer_dim_feedforward=cfg.codecformer_dim_feedforward,
                   context=cfg.context))
    m.load_state_dict(L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05), strict=True)
    m.use_cuda_graphs = True
    m = m.to(DEV, torch.bfloat16).eval()
    yield m
    m.streaming_forever(1)
    m._state = None


@pytest.fixture(scope="module")
def moshi():
    from oracle import moshi_oracle as M
    from rstnet_b200.moshi import LMModel
    m = LMModel(**M.SMALL.reference_kwargs())
    m.load_state_dict(M.synthetic_weights(M.SMALL, seed=5), strict=True)
    return m.to(DEV, torch.bfloat16).eval()


AUDIO = {s: 0.1 * torch.randn(F * TICKS, generator=torch.Generator().manual_seed(40 + i))
         for i, s in enumerate(("me", "argmax", "topk", "plain"))}
MINE = (Sampling(top_p=0.8, top_p_text=0.9, temp=1.0), 77)
OTHERS = {"argmax": (Sampling(use_sampling=False), 3), "topk": (Sampling(top_k=5, temp=1.1), 9), "plain": (None, None)}


def _serve(engine, plan):
    """plan: {session: (admission tick, sampling, seed)}, admitted in the plan's order within a tick; every session pushes
    its own audio for TICKS ticks from its admission.  -> {session: [(tokens, pcm) per tick]}, {session: row}"""
    from rstnet_b200.serve import FrameScheduler
    sch = FrameScheduler(engine, engine.B)
    got, sent, rows = {s: [] for s in plan}, {s: 0 for s in plan}, {}
    last = max(a for a, _, _ in plan.values()) + TICKS
    for t in range(last):
        for s, (a, sp, seed) in plan.items():
            if t == a:
                rows[s] = sch.admit(s) if sp is None and seed is None else sch.admit(s, sampling=sp, seed=seed)
        for s in sch.sessions():
            if sent[s] < TICKS:
                sch.push(s, AUDIO[s][F * sent[s]:F * (sent[s] + 1)])
                sent[s] += 1
        for s, o in sch.tick().items():
            got[s].append(o)
    return got, rows


def _same(a, b):
    assert len(a) == len(b) == TICKS
    for i, ((ta, pa), (tb, pb)) in enumerate(zip(a, b)):
        assert (ta is None) == (tb is None) and (pa is None) == (pb is None), i
        if ta is not None:
            assert torch.equal(ta, tb), i
        if pa is not None:
            assert torch.equal(pa, pb), i


def _plans():
    """the session 'me' in row 0 at tick 0, in row 2 at tick 2, and in row 1 at tick 3, beside sessions with other settings;
    'plain' (no settings, always admitted after a session that brought settings) in rows 2, 3 and 2"""
    o = OTHERS
    return [
        {"me": (0,) + MINE, "argmax": (0,) + o["argmax"], "plain": (1,) + o["plain"]},
        {"argmax": (0,) + o["argmax"], "topk": (0,) + o["topk"], "me": (2,) + MINE, "plain": (2,) + o["plain"]},
        {"topk": (0,) + o["topk"], "me": (3,) + MINE, "plain": (4,) + o["plain"]},
    ]


def _check(runs):
    (g0, r0), (g1, r1), (g2, r2) = runs
    assert (r0["me"], r1["me"], r2["me"]) == (0, 2, 1)
    _same(g0["me"], g1["me"])
    _same(g0["me"], g2["me"])
    # after the switch a session without settings samples with the engine's defaults and key 0, whatever its row / tick
    _same(g0["plain"], g1["plain"])
    _same(g0["plain"], g2["plain"])
    _same(g0["argmax"], g1["argmax"])
    _same(g1["topk"], g2["topk"])
    assert any(p is not None for _, p in g0["me"])


def test_duplex_engine_sessions_with_own_settings(codec, gpt):
    from rstnet_b200.serve import DuplexEngine
    runs = [_serve(DuplexEngine(codec, gpt, 4), plan) for plan in _plans()]
    _check(runs)
    # 'plain' draws as a session given the engine's defaults and seed 0 explicitly
    g, _ = _serve(DuplexEngine(codec, gpt, 4), {"argmax": (0,) + OTHERS["argmax"], "plain": (3, Sampling(), 0)})
    _same(runs[0][0]["plain"], g["plain"])


def test_moshi_engine_sessions_with_own_settings(codec, moshi):
    from rstnet_b200.moshi import LMGen
    from rstnet_b200.serve import MoshiDuplexEngine
    mk = lambda: MoshiDuplexEngine(codec, LMGen(moshi, use_sampling=True, temp=0.8, top_k=250), 4)   # noqa: E731
    runs = [_serve(mk(), plan) for plan in _plans()]
    _check(runs)
    defaults = Sampling(use_sampling=True, temp=0.8, top_k=250, temp_text=0.7, top_k_text=25)
    g, _ = _serve(mk(), {"argmax": (0,) + OTHERS["argmax"], "plain": (3, defaults, 0)})
    _same(runs[0][0]["plain"], g["plain"])
