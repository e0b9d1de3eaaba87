"""CPU tests of `MoshiDuplexEngine`'s host logic (rstnet_b200/serve.py) under `FrameScheduler`, with a fake codec and a
fake LMGen: the decoder's mask is active & valid, a row returns no PCM during its warm-up, released rows are readmitted
with a fresh warm-up."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from rstnet_b200._lib import RstnetError
from rstnet_b200.serve import FrameScheduler, MoshiDuplexEngine

DEP_Q, N_USER, MAX_DELAY = 8, 8, 2


class FakeCodec:
    n_q, codebook_size = N_USER, 2048

    def __init__(self):
        self.masks, self.decode_masks, self.resets = [], [], []

    def streaming_forever(self, B):
        self.B = B

    def reset_streaming(self, streams=None):
        self.resets.append(list(streams))

    def set_active_streams(self, mask):
        self.masks.append(torch.as_tensor(mask).clone())

    def encode(self, pcm):                                  # codes = the first sample of the row's chunk
        return pcm[:, :, :1].round().long().expand(-1, N_USER, -1).contiguous()

    def decode(self, codes):
        self.decode_masks.append(self.masks[-1])
        return codes[:, :1].float().expand(-1, 1, 1920).contiguous()


class FakeLMGen:
    """Per-row step counts with a warm-up of MAX_DELAY steps; the text token is the row's input code + its step count."""

    def __init__(self):
        self.lm_model = SimpleNamespace(device=torch.device("cpu"), num_codebooks=N_USER + DEP_Q + 1, dep_q=DEP_Q)

    def streaming_forever(self, B):
        self.off = np.zeros(B, dtype=np.int64)
        self.act = np.ones(B, dtype=bool)

    def reset_streaming(self, streams=None):
        self.off[list(streams)] = 0

    def set_active_streams(self, mask):
        self.act = torch.as_tensor(mask).numpy() != 0

    def valid_rows(self):
        return self.act & (self.off > MAX_DELAY)

    def step(self, codes):
        self.off += self.act
        if not (self.off > MAX_DELAY).any():
            return None
        tok = codes[:, :1, 0] + torch.from_numpy(self.off)[:, None]
        return tok.expand(-1, DEP_Q + 1)[:, :, None].contiguous()


def test_moshi_engine_host_logic():
    codec, gen = FakeCodec(), FakeLMGen()
    eng = MoshiDuplexEngine(codec, gen, 3)
    sch = FrameScheduler(eng, 3)
    frame = lambda v: torch.full((1920,), float(v))
    got = {"a": [], "b": [], "c": []}
    sch.admit("a")                                           # row 0
    for t in range(7):
        if t == 1:
            sch.admit("b")                                   # row 1
        if t == 5:
            sch.release("a")
            sch.admit("c")                                   # row 0 again, with a fresh warm-up
        for s in sch.sessions():
            if not (s == "b" and t == 3):                    # b sends no audio at tick 3
                sch.push(s, frame(10 * (t + 1)))
        n_dec = len(codec.decode_masks)
        out = sch.tick()
        for s, v in out.items():
            got[s].append(v)
        if len(codec.decode_masks) > n_dec:
            # the decode ran under active & valid, after the encode ran under the active mask
            dec = codec.decode_masks[-1]
            enc = codec.masks[-2]
            assert torch.equal(dec, enc * torch.from_numpy(gen.valid_rows().astype(np.int64)))
        else:
            assert all(v == (None, None) for v in out.values())
    # every session: no PCM (and no tokens) for exactly its first MAX_DELAY ticks
    for s, vs in got.items():
        assert [v[1] is None for v in vs] == [i < MAX_DELAY for i in range(len(vs))], s
        assert all((tk is None) == (p is None) for tk, p in vs)
    assert len(got["a"]) == 5 and len(got["b"]) == 5 and len(got["c"]) == 2
    # tokens of a valid row: its input code + its own step count; PCM = the decoded first code
    tk, pcm = got["a"][2]
    assert int(tk[0]) == 30 + 3 and float(pcm[0]) == float(tk[1])
    tk, pcm = got["b"][2]                                    # b's third step came at tick 4 (no audio at tick 3)
    assert int(tk[0]) == 50 + 3
    assert codec.resets == [[0], [1], [0]]


def test_moshi_engine_rejects():
    with pytest.raises(RstnetError):
        MoshiDuplexEngine(FakeCodec(), FakeLMGen(), 257)
    with pytest.raises(RstnetError):
        MoshiDuplexEngine(FakeCodec(), FakeLMGen(), 2, sample_rate=12345)
    codec = FakeCodec()
    codec.n_q = 4
    with pytest.raises(RstnetError):
        MoshiDuplexEngine(codec, FakeLMGen(), 2)
