"""Continuous batching of ragged corpora through the codec (-m gpu): the tail-fill kernel against a torch restatement,
MimiCodec.encode_many / decode_many against per-clip encode / decode (bit for bit on the fp32 CUDA-core path, by the
margin rule on the tensor cores, and independent of the capacity and of a clip's row and admission step), inputs on
which a plain streaming scope differs from the non-streaming codec, and the offline drivers and CLIs."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import mimi_oracle as O
from oracle import mimi_spec as S
from rstnet_b200 import ops
from rstnet_b200.codec import MimiCodec

pytestmark = pytest.mark.gpu

DEV = "cuda"
FS = 1920
MARGIN = 1e-4
# ends on every side of a frame and of a 24 kHz sample block; 12 s + 17 and 41 s run past the 250-token (10 s) window
LENGTHS = [1, 959, 1919, 1920, 1921, 4000, 7 * FS + 5, 12 * 24000 + 17, 41 * 24000]


@pytest.fixture(scope="module")
def codec(official_weights):
    m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(official_weights, strict=True)
    m = m.to(DEV).eval()
    yield m
    m.streaming_tensor_cores, m.use_cuda_graphs = True, True


def _clips(lengths, seed):
    return [(f"c{i}_{L}", S.synthetic_audio(1, L, seed=seed + i)[0, 0]) for i, L in enumerate(lengths)]


@pytest.fixture(scope="module")
def per_clip(codec):
    """clips, and each clip's own non-streaming encode and decode (B = 1: the fp32 CUDA-core path)."""
    clips = _clips(LENGTHS, 100)
    with torch.no_grad():
        codes = {k: codec.encode(w[None, None].to(DEV))[0].cpu() for k, w in clips}
        wavs = {k: codec.decode(c[None].to(DEV))[0, 0].cpu() for k, c in codes.items()}
    return clips, codes, wavs


# ---------------------------------------------------------------- kernel
def _tail_case(layout, div):
    streams, cps, rows, row0, nrows = 6, 12, 11, 2, 7
    # ceil(valid / div): 0, 1, 3 (mid-range), nrows, clamped to nrows, negative -> 0
    valid = torch.tensor([0, 1, 2 * div + 1, nrows * div, 10 ** 6, -3], dtype=torch.int64)
    if layout == "batch_major":
        batch, C, bs = streams, cps, rows * cps + 4
        pos = lambda s, r, c: s * bs + r * C + c
    else:
        batch, C, bs = 1, streams * cps, 0
        pos = lambda s, r, c: r * C + s * cps + c
    n = (batch - 1) * bs + rows * C + 16           # 16 trailing elements no stream owns
    return streams, cps, row0, nrows, valid, batch, C, bs, pos, n


def _tail_ref(buf, streams, cps, row0, nrows, valid, div, mode, pos):
    ref = buf.clone()
    for s in range(streams):
        k = min(nrows, max(0, -(-int(valid[s]) // div)))
        for r in range(row0 + k, row0 + nrows):
            for c in range(cps):
                ref[pos(s, r, c)] = ref[pos(s, row0 + k - 1, c)] if mode == 1 else 0.0
    return ref


@pytest.mark.parametrize("layout", ["batch_major", "time_major"])
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("div", [1, 4])
def test_rows_fill_tail(layout, mode, div):
    streams, cps, row0, nrows, valid, batch, C, bs, pos, n = _tail_case(layout, div)
    buf = torch.randn(n, generator=torch.Generator().manual_seed(7 * mode + div))
    d = buf.to(DEV)
    ops.rows_fill_tail(d, bs, batch, C, row0, nrows, mode, valid.to(DEV), div, channels_per_stream=cps)
    torch.cuda.synchronize()
    ref = _tail_ref(buf, streams, cps, row0, nrows, valid, div, mode, pos)
    assert torch.equal(d.cpu().view(torch.int32), ref.view(torch.int32))   # the fill, and every other byte untouched


def test_rows_fill_tail_reads_counts_at_replay():
    """One captured launch serves every step: the counts are read from the device tensor when the graph replays."""
    streams, cps, row0, nrows, valid, batch, C, bs, pos, n = _tail_case("time_major", 1)
    buf = torch.randn(n, generator=torch.Generator().manual_seed(3))
    d, v = buf.to(DEV), torch.full((streams,), nrows, dtype=torch.int64, device=DEV)
    ops.rows_fill_tail(d, bs, batch, C, row0, nrows, 0, v, 1, channels_per_stream=cps)   # warm-up: no-op
    torch.cuda.synchronize()
    assert torch.equal(d.cpu(), buf)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.rows_fill_tail(d, bs, batch, C, row0, nrows, 0, v, 1, channels_per_stream=cps)
    v.copy_(valid)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(d.cpu().view(torch.int32), _tail_ref(buf, streams, cps, row0, nrows, valid, 1, 0, pos).view(torch.int32))


def test_rows_fill_tail_refuses_bad_arguments():
    from rstnet_b200._lib import RstnetError
    d, v = torch.zeros(64, device=DEV), torch.zeros(4, dtype=torch.int64, device=DEV)
    with pytest.raises(RstnetError):
        ops.rows_fill_tail(d, 0, 1, 16, 0, 4, 1, v, 1, channels_per_stream=4)    # replicate needs a row before row0
    with pytest.raises(RstnetError):
        ops.rows_fill_tail(d, 0, 1, 16, 1, 3, 0, v, 0, channels_per_stream=4)    # valid_div < 1
    with pytest.raises(RstnetError):
        ops.rows_fill_tail(d, 0, 1, 16, 1, 3, 0, v, 1, channels_per_stream=5)    # C not a multiple of cps


# ---------------------------------------------------------------- exactness on the fp32 CUDA-core path
@pytest.mark.parametrize("capacity", [1, 3, 7])
def test_ffma_encode_decode_many_equal_per_clip_bit_for_bit(codec, per_clip, capacity):
    clips, ref_codes, ref_wavs = per_clip
    codec.streaming_tensor_cores = False
    try:
        got = dict(codec.encode_many(clips, capacity))
        assert sorted(got) == sorted(k for k, _ in clips)
        for key, w in clips:
            assert got[key].dtype == torch.int64 and got[key].shape == (8, math.ceil(w.numel() / FS)), key
            assert torch.equal(got[key], ref_codes[key]), key
        wavs = dict(codec.decode_many(list(ref_codes.items()), capacity))
        for key, c in ref_codes.items():
            assert wavs[key].shape == (FS * c.shape[1],), key
            assert torch.equal(wavs[key].view(torch.int32), ref_wavs[key].view(torch.int32)), key
    finally:
        codec.streaming_tensor_cores = True


def test_empty_items_and_argument_checks(codec):
    out = list(codec.encode_many([("e", torch.zeros(0))], 2))
    assert len(out) == 1 and out[0][0] == "e" and out[0][1].shape == (8, 0)
    out = list(codec.decode_many([("e", torch.zeros(8, 0, dtype=torch.int64))], 2))
    assert out[0][1].shape == (0,)
    with pytest.raises(ValueError):
        list(codec.encode_many([("x", torch.zeros(1, 100))], 2))
    with pytest.raises(ValueError):
        list(codec.decode_many([("x", torch.zeros(8, 3))], 2))
    with pytest.raises(ValueError):
        list(codec.encode_many([], 0))


# ---------------------------------------------------------------- what a plain streaming scope gets wrong
def _plain_streaming_latents(codec, w):
    """latents [frames, 512] of `w` zero-padded to whole frames through a plain streaming(1) scope"""
    T = math.ceil(w.numel() / FS)
    x = torch.zeros(1, 1, T * FS)
    x[0, 0, :w.numel()] = w
    lats = []
    with codec.streaming(1):
        for i in range(T):
            codec.encode(x[..., i * FS:(i + 1) * FS].to(DEV))
            lats.append(codec._stream_state.enc[FS].lat.clone())
    return torch.cat(lats).cpu()


def _batch_latents(codec, w):
    codec.encode(w[None, None].to(DEV))
    eng = codec._eng()
    return next(p for k, p in eng._plans.items() if k[:3] == ("enc", 1, w.numel())).lat.cpu()


def test_plain_streaming_differs_at_clip_end_and_beyond_10s(codec):
    """Why the corpus scope needs the tail fill and the wider rings: through a plain streaming(1) scope, a zero-padded
    clip's last frame and every frame past 250 transformer tokens (10 s) come out differently from `encode`, while the
    frames before agree bit for bit (fp32 CUDA-core path)."""
    codec.streaming_tensor_cores = False
    try:
        with torch.no_grad():
            w = S.synthetic_audio(1, 7 * FS + 5, seed=5)[0, 0]
            s, b = _plain_streaming_latents(codec, w), _batch_latents(codec, w)
            assert torch.equal(s[:-1], b[:-1])
            assert not torch.equal(s[-1], b[-1])          # the encoder's right padding at the clip's end
            w = S.synthetic_audio(1, 12 * 24000, seed=6)[0, 0]   # whole frames: no tail
            s, b = _plain_streaming_latents(codec, w), _batch_latents(codec, w)
            # token 249 (frame 124) is the first whose window holds 250 keys; the ring leaves it 249
            assert torch.equal(s[:124], b[:124])
            assert not torch.equal(s[124:], b[124:])
    finally:
        codec.streaming_tensor_cores = True


# ---------------------------------------------------------------- tensor-core path (default)
def test_tensor_core_many_by_margin_and_capacity_independent(codec, per_clip, official_weights):
    clips, ref_codes, ref_wavs = per_clip
    assert codec.streaming_tensor_cores
    c7 = dict(codec.encode_many(clips, 7))
    c1 = dict(codec.encode_many(list(reversed(clips)), 1))
    flips = 0
    for key, w in clips:
        assert torch.equal(c7[key], c1[key]), key
        bad = (c7[key] != ref_codes[key]).any(dim=0)
        if bool(bad.any()):
            z = O.encode_latent(w[None, None], official_weights)
            margins = O.rvq_margins(z, official_weights).min(dim=0).values.view(-1)[: bad.numel()]
            assert not bool((bad & (margins > MARGIN)).any()), key
            flips += int(bad.sum())
    print(f"tensor-core encode_many: {flips} near-tie frames differ from per-clip encode")
    w7 = dict(codec.decode_many(list(ref_codes.items()), 7))
    w1 = dict(codec.decode_many(list(reversed(list(ref_codes.items()))), 1))
    for key, ref in ref_wavs.items():
        assert torch.equal(w7[key].view(torch.int32), w1[key].view(torch.int32)), key
        peak = max(1.0, float(ref.abs().max()))
        assert float((w7[key] - ref).abs().max()) <= 1e-4 * peak, key


# ---------------------------------------------------------------- offline drivers
def test_tokenize_corpus_equals_encode_many(codec):
    from rstnet_b200 import offline
    from rstnet_b200.audio import Resample
    clips = _clips([4000, 1920, 0, 12345, 100], 300)
    w16 = S.synthetic_audio(1, 8001, seed=9)[0, 0]
    items = clips + [("r16", w16, 16000)]
    toks = offline.tokenize_corpus(codec, items, capacity=3)
    assert set(toks) == {k for k, w in clips if w.numel()} | {"r16"}      # the empty clip is skipped
    y16 = Resample(16000, 24000)(w16.to(DEV)).cpu()
    ref = dict(codec.encode_many([(k, w) for k, w in clips if w.numel()] + [("r16", y16)], 3))
    for k, c in toks.items():
        assert c.dtype == torch.int16 and torch.equal(c, ref[k].to(torch.int16)), k
    assert toks["r16"].shape == (8, math.ceil(math.ceil(8001 * 1.5) / FS))


def test_tokenize_and_reconstruct_cli_with_capacity(codec, official_weights, tmp_path):
    from scipy.io import wavfile
    from rstnet_b200 import offline
    wpath = os.path.join(tmp_path, "w.pt")
    torch.save(official_weights, wpath)
    src = os.path.join(tmp_path, "in")
    os.makedirs(src)
    files = {"a.wav": (24000, 4000), "b.wav": (24000, 1920), "c.wav": (24000, 30000), "d.wav": (16000, 15999), "e.wav": (24000, 0)}
    for i, (name, (sr, L)) in enumerate(files.items()):
        x = S.synthetic_audio(1, L, seed=60 + i)[0, 0] if L else torch.zeros(0)
        wavfile.write(os.path.join(src, name), sr, (x.numpy() * 32767).astype(np.int16))
    scp = os.path.join(tmp_path, "wav.scp")
    with open(scp, "w") as f:
        for name in files:
            f.write(f"{name[0]} {os.path.join(src, name)}\n")
    out = os.path.join(tmp_path, "codes.pt")
    assert offline.main(["tokenize", "--weights", wpath, "--wav-scp", scp, "--output-file", out, "--capacity", "3"]) == 0
    toks = torch.load(out)
    assert set(toks) == {"a", "b", "c", "d"}                  # the empty clip is skipped
    for name, (sr, L) in files.items():
        if L:
            assert toks[name[0]].dtype == torch.int16
            assert toks[name[0]].shape == (8, math.ceil(math.ceil(L * 24000 / sr) / FS)), name
    dst = os.path.join(tmp_path, "out")
    assert offline.main(["reconstruct", "--weights", wpath, "--input", src, "--output", dst, "--capacity", "2"]) == 0
    for name, (sr, L) in files.items():
        rec, rsr = offline.read_wav(os.path.join(dst, name))
        assert rsr == 24000 and rec.numel() == math.ceil(L * 24000 / sr), name
