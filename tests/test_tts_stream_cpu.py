"""CPU tests of streamed TTS (InferenceImp.stream_many, serve.TTSEngine) with a stand-in GPT, codec and delay cache: the
admissions are generate_many's, every utterance's chunks come in order with one codec frame each, the host hands a frame's
chunks out one frame after it ran, and the engine checks its arguments at submit."""
from contextlib import contextmanager

import numpy as np
import pytest
import torch

from rstnet_b200 import infer
from rstnet_b200._lib import RstnetError
from rstnet_b200.infer import InferenceImp, Sampling, TTSChunk
from rstnet_b200.serve import TTSEngine

TEXT_EMPTY, PAD, FS = 128002, 2049, 1920


class FakeGPT:
    """Row r's tokens at its generated frame g are tag * 1000 + g in every codebook (the tag is the utterance's prompt),
    so every code and every PCM sample traces back to the utterance and frame that made it."""
    num_codebooks = 9
    device = torch.device("cpu")

    def __init__(self):
        self.log = []

    @contextmanager
    def streaming(self, B):
        self.B = B
        self.step = np.zeros(B, dtype=np.int64)
        self.active = np.ones(B, dtype=np.int64)
        self.tag = np.zeros(B, dtype=np.int64)
        yield
        self.log.append(("exit",))

    def _get_initial_token(self):
        tok = torch.full([1, 9, 1], 2048, dtype=torch.long)
        tok[:, 0] = 151655
        return tok

    def set_active_streams(self, mask):
        self.active = np.asarray(mask, dtype=np.int64).copy()
        self.log.append(("active", tuple(self.active)))

    def reset_streaming(self, streams=None):
        for s in streams:
            self.step[s] = 0
        self.log.append(("reset", tuple(streams)))

    def prefill_streams(self, prompts):
        self.log.append(("prefill", {s: p.shape[1] for s, p in prompts.items()}))

    def forward_step(self, cur, *, audio_valid, sample_key=None, sampling=None, **kw):
        self.log.append(("step", audio_valid.clone(), self.active.copy(), None if sampling is None else list(sampling),
                         self.step.copy()))
        toks = torch.zeros(self.B, 9, dtype=torch.long)
        for r in range(self.B):
            if self.active[r] and self.step[r] == 0:
                self.tag[r] = int(cur[r, 1, 0])
            if self.active[r]:
                toks[r] = self.tag[r] * 1000 + int(self.step[r])
                self.step[r] += 1
        return toks

    def check_device_errors(self):
        self.log.append(("check",))


class FakeDelay:
    """A torch restatement of the TTS delay of rstnet_lm_delay_cache_out (K 9, delays [0, 0, 1, ..., 1]): after a row's
    generated frame f >= 1, out[1:] is codebook 0 of frame f - 1 and codebooks 1-7 of frame f.  Held rows keep their state."""

    def __init__(self, m, B):
        self.m, self.B = m, B
        self.prev = torch.zeros(B, 9, dtype=torch.long)
        self.off = np.zeros(B, dtype=np.int64)
        self.out = torch.zeros(B, 9, dtype=torch.long)
        self.valid = torch.zeros(B, dtype=torch.long)

    def reset(self, rows):
        for r in rows:
            self.off[r] = 0
            self.valid[r] = 0

    def step(self, toks):
        for b in range(self.B):
            if self.m.active[b]:
                self.out[b, :2] = self.prev[b, :2]
                self.out[b, 2:] = toks[b, 2:]
                self.prev[b] = toks[b]
                self.off[b] += 1
                self.valid[b] = int(self.off[b] > 1)
        return self.out, self.valid


class FakeCodec:
    """decode: pcm[b, k] = code k of row b (k < 8), pcm[b, 8] = the number of decode calls so far, pcm[b, 9] = the row's
    advance flag; records the rows it advanced."""
    codebook_size = 10 ** 7
    frame_size = FS
    sample_rate = 24000

    def __init__(self):
        self.calls, self.log = 0, []

    @contextmanager
    def streaming(self, B, clip_window=False):
        assert clip_window
        self.B = B
        self.mask = torch.zeros(B, dtype=torch.long)
        yield
        self.log.append(("exit",))

    def reset_streaming(self, streams=None):
        self.log.append(("reset", tuple(streams)))

    def set_active_streams(self, mask):
        self.mask = torch.as_tensor(mask).clone()

    def decode(self, codes):
        assert codes.shape == (self.B, 8, 1)
        self.calls += 1
        self.log.append(("decode", tuple(self.mask.tolist())))
        pcm = torch.zeros(self.B, 1, FS)
        pcm[:, 0, :8] = codes[:, :, 0].float()
        pcm[:, 0, 8] = self.calls
        pcm[:, 0, 9] = self.mask.float()
        return pcm


@pytest.fixture(autouse=True)
def fake_delay(monkeypatch):
    monkeypatch.setattr(infer, "_TTSDelay", FakeDelay)


def _utt(P, G, tag):
    seq = torch.full((9, P + G), 7, dtype=torch.long)
    seq[0, P:] = TEXT_EMPTY
    seq[1, :P] = tag
    return torch.cat([seq, torch.full((9, 2), PAD, dtype=torch.long)], 1)


LENS = [(3, 5), (4, 2), (2, 4), (5, 3), (3, 1), (2, 7), (4, 3)]


def _items():
    return [(f"u{i}", _utt(P, G, i + 1)) for i, (P, G) in enumerate(LENS)]


def _imp(m):
    return InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")


def _check_chunks(chunks, codes_ref):
    """every utterance: indices 0 .. G-2 in order, chunk i = codec frame i of its codes, codes on the last chunk only"""
    by_utt = {}
    for c in chunks:
        assert isinstance(c, TTSChunk)
        by_utt.setdefault(c.utt_id, []).append(c)
    assert sorted(by_utt) == sorted(codes_ref)
    for utt, cs in by_utt.items():
        codes = codes_ref[utt]
        G = codes.shape[1] + 1
        assert [c.index for c in cs] == list(range(max(G - 1, 1))), utt
        assert all(c.codes is None for c in cs[:-1]) and torch.equal(cs[-1].codes, codes), utt
        if G == 1:
            assert cs[0].pcm.numel() == 0
            continue
        for c in cs:
            assert c.pcm.dtype == torch.float32 and c.pcm.shape == (FS,)
            assert torch.equal(c.pcm[:8].long(), codes[:, c.index]), (utt, c.index)
            assert c.pcm[9] == 1                  # the row advanced in the codec for this frame


@pytest.mark.parametrize("capacity", [1, 2, 3, 8])
def test_stream_many_chunks_and_admissions_equal_generate_many(capacity):
    m1, m2, codec = FakeGPT(), FakeGPT(), FakeCodec()
    ref = list(_imp(m1).generate_many(_items(), capacity))
    chunks = list(_imp(m2).stream_many(_items(), capacity, codec))
    _check_chunks(chunks, dict(ref))
    # the same scope calls in the same order: admissions, prefills, held rows, candidate tables
    strip = lambda log: [e if e[0] != "step" else ("step", e[1].tolist(), tuple(e[2])) for e in log]
    assert strip(m2.log) == strip(m1.log)
    # utterances complete in generate_many's order
    assert [c.utt_id for c in chunks if c.codes is not None] == [u for u, _ in ref]
    # one codec step per LM frame; the codec resets exactly the admitted rows
    assert codec.calls == sum(1 for e in m1.log if e[0] == "step")
    admitted = [tuple(sorted(e[1])) for e in m1.log if e[0] == "prefill"]
    assert [e[1] for e in codec.log if e[0] == "reset"] == admitted


def test_codec_holds_rows_without_a_frame():
    """a row advances the codec only from its second generated frame on, and never while it is free"""
    m, codec = FakeGPT(), FakeCodec()
    list(_imp(m).stream_many(_items(), 3, codec))
    steps = [e for e in m.log if e[0] == "step"]
    decodes = [e[1] for e in codec.log if e[0] == "decode"]
    assert len(decodes) == len(steps)
    held = 0
    for (_, _, act, _, g), adv in zip(steps, decodes):     # g: the row's generated frames before this step
        for r in range(3):
            assert adv[r] == (1 if act[r] and g[r] >= 1 else 0), (r, act[r], g[r])
            held += not adv[r]
    assert held > 0


def test_stream_many_sampling_and_seeds_as_generate_many():
    m1, m2 = FakeGPT(), FakeGPT()
    sp = {"u2": Sampling(True, 0.5, 5, 0.0, 0.9, 7, 0.0)}
    seeds = {"u1": 11, "u3": 5}
    list(_imp(m1).generate_many(_items(), 3, sampling=sp, seeds=seeds))
    list(_imp(m2).stream_many(_items(), 3, FakeCodec(), sampling=sp, seeds=seeds))
    s1 = [e[3] for e in m1.log if e[0] == "step"]
    s2 = [e[3] for e in m2.log if e[0] == "step"]
    assert s1 == s2 and any(sp["u2"] in s for s in s1)


def test_engine_hands_out_one_frame_behind():
    m, codec = FakeGPT(), FakeCodec()
    ref = dict(_imp(FakeGPT()).generate_many(_items(), 3))
    got = []
    with TTSEngine(_imp(m), codec, 3) as eng:
        for u, s in _items():
            eng.submit(u, s)
        assert eng.pending == len(LENS) and eng.active == 0
        while eng.pending or eng.active:
            before = codec.calls
            out = eng.step()
            ran = codec.calls - before
            # every chunk of this call is from the frame run by the previous call
            for c in out:
                if c.pcm.numel():
                    assert int(c.pcm[8]) == before, (c.utt_id, c.index)
            assert ran in (0, 1)
            got += out
        assert eng.step() == [] and codec.calls == sum(1 for e in m.log if e[0] == "step")
    _check_chunks(got, ref)
    assert m.log[-1] == ("exit",) and ("check",) in m.log


def test_engine_staggered_submissions_reuse_rows_and_idle_steps():
    m, codec = FakeGPT(), FakeCodec()
    items = _items()
    got = []
    with TTSEngine(_imp(m), codec, 2) as eng:
        assert eng.step() == [] and m.log == [("active", (0, 0))] and codec.calls == 0    # nothing to do: no launch
        for t in range(60):
            if t % 3 == 0 and items:
                eng.submit(*items.pop(0))
            got += eng.step()
            if not items and not eng.pending and not eng.active:
                break
        n_steps = sum(1 for e in m.log if e[0] == "step")
        assert eng.step() == [] and sum(1 for e in m.log if e[0] == "step") == n_steps
    assert len({c.utt_id for c in got if c.codes is not None}) == len(LENS)
    # 7 utterances through 2 rows: rows were reused
    assert sum(len(e[1]) for e in m.log if e[0] == "prefill") == len(LENS)
    ref = {}
    for i, (P, G) in enumerate(LENS):
        frames = torch.tensor([[(i + 1) * 1000 + g] * 9 for g in range(G)])
        ref[f"u{i}"] = infer.reverse_delay(frames[:, 1:])
    _check_chunks(got, ref)


def test_engine_argument_checks():
    imp = _imp(FakeGPT())
    for cap in (0, 257, 2.0, True):
        with pytest.raises(RstnetError):
            TTSEngine(imp, FakeCodec(), cap)
    with pytest.raises(RstnetError, match="no paged KV scope"):
        TTSEngine(imp, FakeCodec(), 2, kv_pages=8)
    eng = TTSEngine(imp, FakeCodec(), 2)
    no_gen = torch.full((9, 4), 7, dtype=torch.long)
    with pytest.raises(RstnetError, match="nothing to generate"):
        eng.submit("a", no_gen)
    no_prompt = torch.full((9, 4), 7, dtype=torch.long)
    no_prompt[0] = TEXT_EMPTY
    with pytest.raises(RstnetError, match="no prompt frames"):
        eng.submit("a", no_prompt)
    with pytest.raises(RstnetError):
        eng.submit("a", torch.zeros(8, 4, dtype=torch.long))
    with pytest.raises(RstnetError, match="must be a Sampling"):
        eng.submit("a", _utt(2, 2, 1), sampling={"temp": 1.0})
    with pytest.raises(RstnetError):
        eng.submit("a", _utt(2, 2, 1), seed="1")
    eng.submit("a", _utt(2, 2, 1))
    with pytest.raises(RstnetError, match="already queued"):
        eng.submit("a", _utt(2, 2, 1))
    assert eng.pending == 1
    eng.close()
    with pytest.raises(RstnetError, match="closed"):
        eng.step()
    with pytest.raises(RstnetError, match="closed"):
        eng.submit("b", _utt(2, 2, 1))
    bad = InferenceImp(None, FakeGPT(), "sampling", 0.7, 25, 0.8, 30, "ASR")
    with pytest.raises(NotImplementedError):
        TTSEngine(bad, FakeCodec(), 2)


def test_stream_many_argument_checks():
    imp = _imp(FakeGPT())
    for cap in (0, 257):
        with pytest.raises(RstnetError):
            next(imp.stream_many(_items(), cap, FakeCodec()))
    with pytest.raises(RstnetError, match="must be a Sampling"):
        next(imp.stream_many(_items(), 2, FakeCodec(), sampling={"u0": 3}))
    with pytest.raises(RstnetError, match="no paged KV scope"):
        next(imp.stream_many(_items(), 2, FakeCodec(), kv_pages=4))


def test_synthesize_stream_parser():
    from rstnet_b200 import offline
    a = offline.build_parser().parse_args(["synthesize", "--input", "i", "--config", "c", "--checkpoint", "k",
                                           "--output-file", "o", "--wav-dir", "w", "--stream"])
    assert a.stream
    a = offline.build_parser().parse_args(["synthesize", "--input", "i", "--config", "c", "--checkpoint", "k", "--output-file", "o"])
    assert not a.stream
