"""Streamed TTS on the GPU (-m gpu): InferenceImp.stream_many and serve.TTSEngine against generate_many (codes) and
MimiCodec.decode of those codes (PCM), the codec's clip_window streaming scope, and `offline synthesize --stream`."""
import dataclasses
import json
import os

import pytest
import torch

from oracle import lm_oracle as L
from rstnet_b200._lib import RstnetError
from rstnet_b200.codec import MimiCodec
from rstnet_b200.infer import InferenceImp
from rstnet_b200.lm import GPT, Config, Sampling
from rstnet_b200.serve import TTSEngine

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
BF = torch.bfloat16
TEXT_EMPTY, FS = 128002, 1920


@pytest.fixture(scope="module")
def small_lm():
    """L.SMALL (context 16, block_size 64) as in test_tts_batch_gpu.py."""
    cfg = L.SMALL
    w32 = L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05)
    m = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                   intermediate_size=cfg.intermediate_size, norm_eps=cfg.norm_eps, padded_vocab_size=cfg.padded_vocab_size,
                   audio_card=cfg.audio_card, n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim,
                   codecformer_heads=cfg.codecformer_heads, codecformer_layers=cfg.codecformer_layers,
                   codecformer_dim_feedforward=cfg.codecformer_dim_feedforward, context=cfg.context))
    m.load_state_dict(w32, strict=True)
    m.use_cuda_graphs = True
    return m.to(DEV, BF).eval(), w32


@pytest.fixture(scope="module")
def codec(official_weights):
    m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(official_weights, strict=True)
    m = m.to(DEV).eval()
    m.streaming_tensor_cores, m.use_cuda_graphs = True, True
    return m


def _corpus(n, seed, pmax=20, gmax=12):
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        P = int(torch.randint(3, pmax + 1, (1,), generator=g))
        G = int(torch.randint(1, gmax + 1, (1,), generator=g)) if i else 1     # utterance 0 generates one frame only
        seq = torch.randint(0, 2048, (9, P + G), generator=g)
        seq[0, :P] = torch.randint(0, 1000, (P,), generator=g)
        seq[0, P:] = TEXT_EMPTY
        if i % 3 == 0:                                          # trailing pad frames are stripped
            seq = torch.cat([seq, torch.full((9, 2), 2049)], 1)
        out.append((f"utt{i}", seq))
    return out


def _imp(m):
    return InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")


def _collect(chunks):
    """-> {utt: (pcm [1920 * (G - 1)], codes)}, checking that every utterance's indices run 0 .. G - 2 without gaps"""
    parts, out = {}, {}
    for c in chunks:
        assert c.utt_id not in out, c.utt_id
        parts.setdefault(c.utt_id, []).append(c)
        if c.codes is not None:
            cs = parts.pop(c.utt_id)
            n = c.codes.shape[1]
            assert [x.index for x in cs] == list(range(max(n, 1))), c.utt_id
            assert all(x.codes is None for x in cs[:-1]) and c.codes.device.type == "cpu"
            pcm = torch.cat([x.pcm for x in cs])
            assert pcm.dtype == torch.float32 and pcm.numel() == FS * n
            out[c.utt_id] = (pcm, c.codes)
    assert not parts
    return out


def _decode(codec, codes):
    """whole-utterance decode; ids 2048 / 2049 clamped as the codec's gather does (without its error flag)"""
    if codes.shape[1] == 0:
        return torch.zeros(0)
    return codec.decode(codes.clamp(max=2047)[None].to(DEV))[0, 0].cpu()


def _close(pcm, dec):
    """within 1e-4 x peak of the whole-utterance decode (the rule of decode_many on the tensor cores)"""
    if not dec.numel():
        return pcm.numel() == 0
    return pcm.numel() == dec.numel() and float((pcm - dec).abs().max()) <= 1e-4 * max(1.0, float(dec.abs().max()))


def _reference(imp, corpus, cap, **kw):
    return {u: c.cpu() for u, c in imp.generate_many(((u, s.to(DEV)) for u, s in corpus), cap, **kw)}


def test_stream_many_fp32_pcm_bit_exact(small_lm, codec):
    m, _ = small_lm
    imp = _imp(m)
    corpus = _corpus(10, 3)
    codec.streaming_tensor_cores = False
    try:
        for cap in (1, 3, 7):
            ref = _reference(imp, corpus, cap)
            got = _collect(imp.stream_many(((u, s.to(DEV)) for u, s in corpus), cap, codec))
            assert sorted(got) == sorted(ref)
            for u, (pcm, codes) in got.items():
                assert torch.equal(codes, ref[u]), (cap, u)
                assert torch.equal(pcm.view(torch.int32), _decode(codec, codes).view(torch.int32)), (cap, u)
    finally:
        codec.streaming_tensor_cores = True


def test_stream_many_tensor_cores_by_margin_and_order_independent(small_lm, codec):
    m, _ = small_lm
    imp = _imp(m)
    corpus = _corpus(12, 4)
    assert codec.streaming_tensor_cores
    a = _collect(imp.stream_many(corpus, 3, codec))
    b = _collect(imp.stream_many(list(reversed(corpus)), 7, codec))
    ref = _reference(imp, corpus, 3)
    for u, (pcm, codes) in a.items():
        assert torch.equal(codes, ref[u]) and torch.equal(b[u][1], ref[u]), u
        assert torch.equal(pcm.view(torch.int32), b[u][0].view(torch.int32)), u
        assert _close(pcm, _decode(codec, codes)), u


def test_stream_many_sampling_seeds_and_short_pool(small_lm, codec):
    m, _ = small_lm
    imp = _imp(m)
    corpus = _corpus(9, 8)
    sampling = {"utt2": Sampling(True, 0.9, 5, 0.0, 1.1, 10, 0.0), "utt5": Sampling(False, 0.7, 25, 0.0, 0.8, 30, 0.0),
                "utt7": Sampling(True, 0.7, 25, 0.0, 0.8, 0, 0.9)}
    seeds = {u: 100 + i for i, (u, _) in enumerate(corpus)}
    stats = {}
    ref = {u: c.cpu() for u, c in imp.generate_many(corpus, 4, seeds=seeds, sampling=sampling, kv_pages=2, stats=stats)}
    assert stats["wait_frames"] > 0            # two pages for four rows: admissions waited
    got = _collect(imp.stream_many(corpus, 4, codec, seeds=seeds, sampling=sampling, kv_pages=2))
    assert [u for u in got] == [u for u in ref]     # the same completion order
    for u, (pcm, codes) in got.items():
        assert torch.equal(codes, ref[u]), u


def test_stream_many_capacity_above_128(small_lm, codec):
    m, _ = small_lm
    imp = _imp(m)
    corpus = _corpus(150, 9, pmax=8, gmax=5)
    ref = _reference(imp, corpus, 130)
    got = _collect(imp.stream_many(corpus, 130, codec))
    assert sorted(got) == sorted(ref)
    for u in ("utt1", "utt64", "utt129", "utt149"):
        assert _close(got[u][0], _decode(codec, got[u][1])), u
    for u, (_, codes) in got.items():
        assert torch.equal(codes, ref[u]), u


def test_engine_staggered_reuse_and_errors(small_lm, codec):
    m, _ = small_lm
    imp = _imp(m)
    corpus = _corpus(7, 11)
    ref = _reference(imp, corpus, 2)
    with pytest.raises(RstnetError):
        TTSEngine(imp, codec, 0)
    with pytest.raises(RstnetError):
        TTSEngine(imp, codec, 257)
    chunks, todo = [], list(corpus)
    with TTSEngine(imp, codec, 2) as eng:
        assert eng.step() == []
        bad = torch.full((9, 5), 3)
        with pytest.raises(RstnetError, match="nothing to generate"):
            eng.submit("bad", bad)
        t = 0
        while todo or eng.pending or eng.active:
            if todo and t % 4 == 0:
                eng.submit(*todo.pop(0))
            chunks += eng.step()
            t += 1
        assert eng.step() == []
    got = _collect(chunks)
    assert sorted(got) == sorted(ref)
    for u, (pcm, codes) in got.items():
        assert torch.equal(codes, ref[u]), u
        assert _close(pcm, _decode(codec, codes)), u
    # the engine's scopes are closed: generate_many runs again on the same model
    assert torch.equal(_reference(imp, corpus[:2], 2)["utt1"], ref["utt1"])


def test_clip_window_stream_equals_decode_past_the_window(codec):
    """140 frames (280 decoder transformer tokens, past the 250-token window) one frame per step: with clip_window the
    stream is decode() of the whole clip bit for bit (fp32 path); the reference's ring (clip_window False) is not."""
    codes = torch.randint(0, 2048, (1, 8, 140), generator=torch.Generator().manual_seed(3)).to(DEV)
    codec.streaming_tensor_cores = False
    try:
        ref = codec.decode(codes)[0, 0]
        outs = {}
        for cw in (True, False):
            with codec.streaming(1, clip_window=cw):
                outs[cw] = torch.cat([codec.decode(codes[:, :, t:t + 1])[0, 0] for t in range(140)])
        assert torch.equal(outs[True].view(torch.int32), ref.view(torch.int32))
        assert not torch.equal(outs[False], ref)
    finally:
        codec.streaming_tensor_cores = True


def test_synthesize_stream_cli(small_lm, official_weights, tmp_path):
    from scipy.io import wavfile
    from rstnet_b200 import offline
    m, w32 = small_lm
    (tmp_path / "gpt.json").write_text(json.dumps(dataclasses.asdict(m.config)))
    torch.save({"model": {"module." + k: v for k, v in w32.items()}}, tmp_path / "ckpt.pt")
    torch.save(official_weights, tmp_path / "codec.pt")
    torch.save(dict(_corpus(6, 13)), tmp_path / "corpus.pt")
    common = ["synthesize", "--input", str(tmp_path / "corpus.pt"), "--config", str(tmp_path / "gpt.json"), "--checkpoint",
              str(tmp_path / "ckpt.pt"), "--capacity", "4", "--device", "cuda:0", "--codec-weights", str(tmp_path / "codec.pt")]
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    # the same file name in both runs: torch.save names the archive's records after it
    assert offline.main(common + ["--output-file", str(tmp_path / "a" / "codes.pt"), "--wav-dir", str(tmp_path / "wa")]) == 0
    from rstnet_b200 import _lib
    _lib.lib().rstnet_device_error_flags(1)    # the plain run's decode flags ids 2048 / 2049; clear before the next run
    assert offline.main(common + ["--output-file", str(tmp_path / "b" / "codes.pt"), "--wav-dir", str(tmp_path / "wb"),
                                  "--stream"]) == 0
    assert (tmp_path / "a" / "codes.pt").read_bytes() == (tmp_path / "b" / "codes.pt").read_bytes()
    names = sorted(os.listdir(tmp_path / "wa"))
    assert names and names == sorted(os.listdir(tmp_path / "wb"))
    for n in names:
        a, b = wavfile.read(tmp_path / "wa" / n)[1], wavfile.read(tmp_path / "wb" / n)[1]
        assert a.shape == b.shape, n
