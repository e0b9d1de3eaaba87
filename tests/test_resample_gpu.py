"""GPU resampling (-m gpu): rstnet_resample_f32 / rstnet_b200.audio against the float64 sum of its own fp32 operands and
the torchaudio goldens, the streaming form against the batch form, and the offline drivers and the duplex engine at
client rates other than 24 kHz.  Reads only the goldens and the CPU restatement (tests/resample_oracle.py)."""
import math
import os

import numpy as np
import pytest
import torch

import resample_oracle as R
from oracle import mimi_oracle as O
from oracle import mimi_spec as S
from rstnet_b200 import _lib, audio

pytestmark = pytest.mark.gpu

DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
MARGIN = 1e-4


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "resample.npz"))


def _cases(g, key):
    for name in g[f"{key}__cases"]:
        base = f"{key}__{name}"
        rows, L = (int(v) for v in str(name)[1:].split("_L"))
        x = R.seeded_input(rows, L, int(g[f"{base}__seed"]))
        assert R.sha256(x) == str(g[f"{base}__x_sha256"])
        yield x, torch.from_numpy(g[f"{base}__y"])


def _check_bound(x2d, y, t, golden_y=None):
    """|y - y64| <= S_p u sum|x h| (and, against torchaudio, + K u sum|x h|); returns (worst ratio, bit-equal fraction)"""
    y64, mag = R.run_sums64(x2d, t.taps, t.start, t.o, t.n, -t.width, y.shape[-1])
    runs = (t.taps != 0).sum(1).double()
    sp = runs[torch.arange(y.shape[-1]) % t.n]
    y = y.double().reshape(y64.shape)
    bound = sp * U * mag + 1e-45
    err = (y - y64).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    worst, eq = float((err / bound).max()), 1.0
    if golden_y is not None:
        gy = golden_y.double().reshape(y64.shape)
        gb = (sp + t.K) * U * mag + 1e-45
        gerr = (y - gy).abs()
        assert bool((gerr <= gb).all()), float((gerr / gb).max())
        worst = max(worst, float((gerr / gb).max()))
        eq = float((y == gy).double().mean())
    return worst, eq


@pytest.mark.parametrize("pair", R.PAIRS)
def test_batch_form_per_element_bound(golden, pair):
    key = "%d_%d" % pair
    rs = audio.Resample(*pair)
    t = rs.table
    worst, eqs = 0.0, []
    for x, gy in _cases(golden, key):
        y = rs(x.to(DEV)).cpu()
        assert y.shape == gy.shape
        w, eq = _check_bound(x, y, t, gy)
        worst, eqs = max(worst, w), eqs + [eq]
    # leading dims [2, 3, L], on a length that is not a multiple of o
    L = int(0.05 * pair[0]) + 5
    x = R.seeded_input(6, L, 77).view(2, 3, L)
    y = rs(x.to(DEV)).cpu()
    assert y.shape == (2, 3, math.ceil(t.n * L / t.o))
    assert torch.equal(y.view(6, -1), rs(x.view(6, L).to(DEV)).cpu())
    worst = max(worst, _check_bound(x.view(6, L), y.view(6, -1), t, R.resample(x, *pair).view(6, -1))[0])
    print(f"{key}: worst error / bound {worst:.3f}; bit-equal to torchaudio {min(eqs):.4f}..{max(eqs):.4f}")


def test_canaries_and_strided_rows():
    rs = audio.Resample(44100, 24000)
    t = rs.table
    L, rows = 4411, 3
    out_len = math.ceil(t.n * L / t.o)
    x = torch.zeros(rows, L + 100, device=DEV)
    x[:, :L] = R.seeded_input(rows, L, 3).to(DEV)
    x[:, L:] = float("nan")                                      # past x_len: must never be read
    out = torch.full((rows, out_len + 37), float("nan"), device=DEV)
    taps, start = t.taps.to(DEV), t.start.to(DEV)
    _lib.check(_lib.lib().rstnet_resample_f32(x.data_ptr(), L + 100, L, -t.width, taps.data_ptr(), start.data_ptr(), t.n, t.o,
                                              t.S, t.start_max, out.data_ptr(), out_len + 37, out_len, rows,
                                              torch.cuda.current_stream().cuda_stream), "resample")
    torch.cuda.synchronize()
    assert bool(out[:, out_len:].isnan().all())                 # canaries after every row
    assert torch.equal(out[:, :out_len], rs(x[:, :L].contiguous()))
    assert not bool(out[:, :out_len].isnan().any())


def test_sum_order_is_increasing_taps():
    """The kernel's sum is one fmaf chain from +0 in increasing tap order.  With power-of-two taps and inputs of the form
    k * 2^e every product and every partial sum is exact in float64, so a float64 add followed by a float32 rounding is
    exactly fmaf; the magnitudes span 2^0..2^26, so another order (or a missing tap) rounds differently."""
    g = torch.Generator().manual_seed(5)
    n, o, S, L, rows = 3, 2, 5, 4001, 4
    start = torch.tensor([0, 1, 2], dtype=torch.int32)
    taps = (2.0 ** torch.randint(-1, 2, (n, S), generator=g)) * (torch.randint(0, 2, (n, S), generator=g) * 2 - 1)
    taps = taps.float()
    x = (torch.randint(-4, 5, (rows, L), generator=g) * 2.0 ** torch.randint(0, 27, (rows, L), generator=g)).float()
    out_len = math.ceil(n * L / o)
    acc = torch.zeros(rows, out_len, dtype=torch.float32)
    q = torch.arange(out_len)
    j, p = q // n, q % n
    for i in range(S):
        t = j * o - 4 + start.long()[p] + i
        xv = torch.where((t >= 0) & (t < L), x[:, t.clamp(0, L - 1)], torch.zeros(()))
        acc = (acc.double() + xv.double() * taps[p, i].double()).float()
    xd, out = x.to(DEV), torch.empty(rows, out_len, device=DEV)
    td, sd = taps.to(DEV), start.to(DEV)
    _lib.check(_lib.lib().rstnet_resample_f32(xd.data_ptr(), L, L, -4, td.data_ptr(), sd.data_ptr(), n, o, S, 2, out.data_ptr(),
                                              out_len, out_len, rows, torch.cuda.current_stream().cuda_stream), "resample")
    assert torch.equal(out.cpu(), acc)


def test_identity_and_rejections():
    x = torch.randn(2, 100, device=DEV)
    assert audio.Resample(24000, 24000)(x) is x
    with pytest.raises(_lib.RstnetError, match="CUDA"):
        audio.Resample(16000, 24000)(x.cpu())
    with pytest.raises(_lib.RstnetError, match="float32"):
        audio.Resample(16000, 24000)(x.double())
    with pytest.raises(_lib.RstnetError, match="integer"):
        audio.Resample(16000.5, 24000)
    s = audio.StreamingResampler(16000, 24000, 2, DEV)
    with pytest.raises(_lib.RstnetError, match="multiple"):
        s(torch.zeros(2, 3, device=DEV))
    with pytest.raises(_lib.RstnetError):
        s(torch.zeros(2, 4, device=DEV, dtype=torch.float64))


def _stream(s, x, chunk):
    return torch.cat([s(x[:, i:i + chunk]).clone() for i in range(0, x.shape[1], chunk)], dim=1)


@pytest.mark.parametrize("pair", R.PAIRS)
def test_streaming_equals_batch(pair):
    orig, new = pair
    o, n, _ = R.reduced(orig, new)
    B = 256
    D = R.delay_blocks(orig, new)
    for chunk in (orig * 2 // 25, 5 * o if o > 1 else 37):
        nch = 4
        x = R.seeded_input(B, chunk * nch, 11 + chunk).to(DEV)
        s = audio.StreamingResampler(orig, new, B, DEV)
        got = _stream(s, x, chunk)
        z = torch.cat([torch.zeros(B, D * o, device=DEV), x], dim=1)
        ref = audio.Resample(orig, new)(z)[:, : got.shape[1]]
        assert got.shape[1] == chunk * nch // o * n
        assert torch.equal(got, ref), (pair, chunk)
    # reset of row 5 mid-run; row 9 held for one call
    chunk = orig * 2 // 25
    x = R.seeded_input(B, chunk * 5, 99).to(DEV)
    s = audio.StreamingResampler(orig, new, B, DEV)
    ref_all = _stream(audio.StreamingResampler(orig, new, B, DEV), x, chunk)
    outs = [s(x[:, :chunk]).clone(), s(x[:, chunk:2 * chunk]).clone()]
    s.reset([5])
    mask = torch.ones(B, dtype=torch.int64)
    mask[9] = 0
    s.set_active(mask)
    outs.append(s(x[:, 2 * chunk:3 * chunk]).clone())
    s.set_active(None)
    row9 = torch.arange(B, device=DEV)[:, None] == 9                # the held row resumes with the chunk it missed
    outs.append(s(torch.where(row9, x[:, 2 * chunk:3 * chunk], x[:, 3 * chunk:4 * chunk])).clone())
    got = torch.cat(outs, 1)
    others = [r for r in range(B) if r not in (5, 9)]
    assert torch.equal(got[others], ref_all[others, : got.shape[1]])
    fresh = _stream(audio.StreamingResampler(orig, new, 1, DEV), x[5:6, 2 * chunk:4 * chunk], chunk)
    k = chunk // o * n
    assert torch.equal(got[5, 2 * k:], fresh[0])                   # row 5 restarted as a fresh stream
    assert torch.equal(got[9, :2 * k], ref_all[9, :2 * k])        # row 9: the held call left no trace
    assert torch.equal(got[9, 3 * k:], ref_all[9, 2 * k:3 * k])


# ---------------------------------------------------------------- offline drivers and serving


@pytest.fixture(scope="module")
def codec(official_weights):
    from rstnet_b200.codec import MimiCodec
    m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(official_weights, strict=True)
    return m.to(DEV).eval()


def test_offline_tokenize_at_other_rates(official_weights, codec, golden, tmp_path):
    from rstnet_b200 import offline
    items, refs = [], {}
    for orig, L in ((16000, 16000), (44100, 22050)):
        x = S.synthetic_audio(1, L, seed=int(golden[f"clip{orig}__seed"]))[0, 0]
        assert R.sha256(x) == str(golden[f"clip{orig}__x_sha256"])
        y24 = torch.from_numpy(golden[f"clip{orig}__y24k"])
        items.append((f"c{orig}", x, orig))
        refs[f"c{orig}"] = y24
    toks = offline.tokenize_utterances(codec, items)
    for utt, y24 in refs.items():
        with torch.no_grad():
            ref = codec.encode(y24[None, None].to(DEV)).to(torch.int16).cpu()[0]
            margins = O.rvq_margins(O.encode_latent(y24[None, None], official_weights), official_weights).min(dim=0).values
        assert toks[utt].shape == ref.shape == (8, math.ceil(y24.numel() / 1920))
        bad = (toks[utt] != ref).any(dim=0)
        assert not bool((bad & (margins.view(-1)[: bad.numel()] > MARGIN)).any()), utt
    # 24 kHz: with or without the rate, the same batches and the same codes
    clips = [(f"u{i}", S.synthetic_audio(1, L, seed=40 + i)[0, 0]) for i, L in enumerate([3840, 3840, 5000])]
    a = offline.tokenize_utterances(codec, clips, batch_size=2)
    b = offline.tokenize_utterances(codec, [(u, w, 24000) for u, w in clips], batch_size=2)
    assert all(torch.equal(a[k], b[k]) for k in a)
    # reconstruct: a 16 kHz wav comes back at 24 kHz, ceil(1.5 L) samples
    src, dst = os.path.join(tmp_path, "in"), os.path.join(tmp_path, "out")
    os.makedirs(src)
    from scipy.io import wavfile
    pcm = (0.5 * items[0][1] / items[0][1].abs().max() * 32767).to(torch.int16).numpy()
    wavfile.write(os.path.join(src, "a.wav"), 16000, pcm[:15999])
    assert offline.reconstruct_directory(codec, src, dst) == 1
    rec, sr = offline.read_wav(os.path.join(dst, "a.wav"))
    assert sr == 24000 and rec.numel() == math.ceil(1.5 * 15999)


def _small_lm():
    from oracle import lm_oracle as L
    from rstnet_b200.lm import GPT, Config
    cfg = L.SMALL
    lm = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                    intermediate_size=cfg.intermediate_size, padded_vocab_size=cfg.padded_vocab_size, audio_card=cfg.audio_card,
                    n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim, codecformer_heads=cfg.codecformer_heads,
                    codecformer_layers=cfg.codecformer_layers, codecformer_dim_feedforward=cfg.codecformer_dim_feedforward,
                    context=cfg.context))
    lm.load_state_dict(L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05), strict=True)
    return lm.to(DEV, torch.bfloat16).eval()


@pytest.fixture(scope="module")
def lm():
    m = _small_lm()
    yield m
    m.streaming_forever(1)
    m._state = None


def _client_audio(rate, rows, frames, seed):
    F = rate * 2 // 25
    return R.seeded_input(rows, F * frames, seed) * 0.3, F


@pytest.mark.parametrize("rate", [16000, 48000])
def test_duplex_engine_at_client_rate_equals_resampled_24k_engine(codec, lm, rate):
    from rstnet_b200.serve import DuplexEngine
    codec.use_cuda_graphs, codec.streaming_tensor_cores = True, True
    B, ticks = 4, 6
    x, F = _client_audio(rate, B, ticks, 3)
    eng = DuplexEngine(codec, lm, B, use_sampling=False, sample_rate=rate)
    got = [eng.step({r: x[r, i * F:(i + 1) * F] for r in range(B)}, list(range(B))) for i in range(ticks)]
    up = audio.StreamingResampler(rate, 24000, B, DEV)
    down = audio.StreamingResampler(24000, rate, B, DEV)
    eng24 = DuplexEngine(codec, lm, B, use_sampling=False)
    for i in range(ticks):
        x24 = up(x[:, i * F:(i + 1) * F].to(DEV)).cpu()
        o24 = eng24.step({r: x24[r] for r in range(B)}, list(range(B)))
        pcm = down(torch.stack([o24[r][1] for r in range(B)]).to(DEV)).cpu()
        for r in range(B):
            assert torch.equal(got[i][r][0], o24[r][0]), (i, r)
            assert got[i][r][1].shape == (F,) and torch.equal(got[i][r][1], pcm[r]), (i, r)
    codec._stream_state = None


def test_frame_scheduler_with_duplex_engine_at_16k(codec, lm):
    """The session-independence check of the 24 kHz scheduler test at a 16 kHz client rate: late admission, a held tick
    and a release leave every session's tokens and PCM exactly as if it were alone."""
    from rstnet_b200.serve import DuplexEngine, FrameScheduler
    codec.use_cuda_graphs, codec.streaming_tensor_cores = True, True
    audio16, F = _client_audio(16000, 3, 6, 55)
    fr = lambda s, i: audio16[s, i * F:(i + 1) * F]

    def session_alone(s):
        sch = FrameScheduler(DuplexEngine(codec, lm, 4, use_sampling=False, sample_rate=16000), 4)
        sch.admit("x")
        out = []
        for i in range(6):
            sch.push("x", fr(s, i))
            out.append(sch.tick()["x"])
        return out

    alone = [session_alone(s) for s in range(3)]
    eng = DuplexEngine(codec, lm, 4, use_sampling=False, sample_rate=16000)
    sch = FrameScheduler(eng, 4)
    sch.admit("A")
    got = {"A": [], "B": [], "C": []}
    nxt = {"A": 0, "B": 0, "C": 0}
    src = {"A": 0, "B": 1, "C": 2}
    for tick in range(9):
        if tick == 1:
            sch.admit("B")
        if tick == 3:
            sch.admit("C")
        for name in list(sch.sessions()):
            if name == "B" and tick == 4:
                continue
            if nxt[name] < 6:
                sch.push(name, fr(src[name], nxt[name]))
                nxt[name] += 1
        for name, o in sch.tick().items():
            got[name].append(o)
        if tick == 6:
            sch.release("A")
    for name in ("A", "B", "C"):
        assert len(got[name]) == 6
        for (t_a, p_a), (t_b, p_b) in zip(got[name], alone[src[name]]):
            assert p_a.shape == (F,) and torch.equal(t_a, t_b) and torch.equal(p_a, p_b), name
    codec._stream_state = None


def test_duplex_engine_capacity_256_at_48k(codec, lm):
    from rstnet_b200.serve import DuplexEngine
    codec.use_cuda_graphs, codec.streaming_tensor_cores = True, True
    B = 256
    x, F = _client_audio(48000, B, 2, 8)
    eng = DuplexEngine(codec, lm, B, use_sampling=False, sample_rate=48000)
    for i in range(2):
        out = eng.step({r: x[r, i * F:(i + 1) * F] for r in range(B)}, list(range(B)))
        assert len(out) == B and all(o[1].shape == (F,) and bool(torch.isfinite(o[1]).all()) for o in out.values())
    codec._stream_state = None
