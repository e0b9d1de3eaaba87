"""CPU tests of InferenceImp.generate_many's host logic (rstnet_b200/infer.py) with a fake GPT: admission order, row
reuse, completion order, the per-row candidate table, and the C ABI of the ragged prefill / per-row sampling."""
import os
import random
import re
from contextlib import contextmanager

import numpy as np
import pytest
import torch

from rstnet_b200 import _lib
from rstnet_b200.infer import InferenceImp, candidate_counts, reverse_delay

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TEXT_EMPTY, PAD = 128002, 2049


def reference_rule(pre_gen_len, minlen, g_idx):
    """infer_no_streaming.py:264-283, transcribed branch by branch (2049: sample_token_audio, 2048: ..._2048)."""
    g_len = pre_gen_len + g_idx
    out = []
    for l_idx in range(8):
        if g_len == pre_gen_len:
            out.append(2049)
        elif l_idx > 0 and g_len > minlen:
            out.append(2049)
        else:
            out.append(2048)
    return out


def test_candidate_counts_match_reference_rule():
    rng = random.Random(5)
    for _ in range(2000):
        P, G = rng.randint(1, 200), rng.randint(1, 300)
        g = rng.randrange(G)
        assert candidate_counts(P, G, g) == reference_rule(P, G, g), (P, G, g)


class FakeGPT:
    """Records the scope calls; row r's tokens at a frame are (utterance tag, its frame index) so every yielded code can
    be traced back to the row and frame that made it."""
    num_codebooks = 9
    device = torch.device("cpu")

    def __init__(self):
        self.log = []

    @contextmanager
    def streaming(self, B):
        self.B = B
        self.pos = np.zeros(B, dtype=np.int64)
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
            self.pos[s] = 0
            self.step[s] = 0
        self.log.append(("reset", tuple(streams)))

    def prefill_streams(self, prompts):
        for s, p in prompts.items():
            assert p.shape[0] == 9
            self.pos[s] += p.shape[1]
        self.log.append(("prefill", {s: p.shape[1] for s, p in prompts.items()}))

    def forward_step(self, cur, *, audio_valid, sample_key=None, **kw):
        assert cur.shape == (self.B, 9, 1) and audio_valid.shape == (self.B, 8)
        self.log.append(("step", audio_valid.clone(), self.active.copy()))
        toks = torch.zeros(self.B, 9, dtype=torch.long)
        for r in range(self.B):
            if self.active[r] and self.step[r] == 0:
                self.tag[r] = int(cur[r, 1, 0])   # an admitted row starts from its last prompt frame, which names it
            if self.active[r]:
                toks[r] = torch.tensor([self.tag[r] * 1000 + self.step[r]] * 9)
                self.step[r] += 1
                self.pos[r] += 1
        return toks

    def check_device_errors(self):
        pass


def _utt(P, G, tag):
    seq = torch.full((9, P + G), 7, dtype=torch.long)
    seq[0, P:] = TEXT_EMPTY
    seq[1, :P] = tag
    return torch.cat([seq, torch.full((9, 3), PAD, dtype=torch.long)], 1)   # trailing pad frames are stripped


def test_admission_row_reuse_and_completion_order():
    lens = [(3, 5), (4, 2), (2, 4), (5, 3), (3, 1)]
    items = [(f"u{i}", _utt(P, G, i + 1)) for i, (P, G) in enumerate(lens)]
    m = FakeGPT()
    imp = InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, "TTS")
    out = list(imp.generate_many(items, capacity=2))
    # u0 (G 5) and u1 (G 2) start together; u1 ends after frame 2, u2 takes its row (frames 3-6); u0 ends after frame 5,
    # u3 takes row 0 (frames 6-8); u2 ends after frame 6, u4 takes row 1 (frame 7)
    assert [u for u, _ in out] == ["u1", "u0", "u2", "u4", "u3"]
    resets = [e[1] for e in m.log if e[0] == "reset"]
    assert resets == [(0, 1), (1,), (1,), (0,), (0,), (1,), (1,), (1,), (0,)]
    prefills = [e[1] for e in m.log if e[0] == "prefill"]
    # the init frame + all prompt frames but the last
    assert prefills == [{0: 3, 1: 4}, {1: 2}, {0: 5}, {1: 3}]
    for (utt, codes), (i, (P, G)) in zip(sorted(out), enumerate(lens)):
        tag = int(utt[1:]) + 1
        frames = torch.tensor([[tag * 1000 + g] * 9 for g in range(G)])
        assert torch.equal(codes, reverse_delay(frames[:, 1:])), utt
    steps = [e for e in m.log if e[0] == "step"]
    assert len(steps) == 8
    assert [tuple(a) for _, _, a in steps][-1] == (1, 0)          # the last frame holds the empty row
    assert m.log[-1] == ("exit",)


def test_candidate_table_per_row():
    rng = random.Random(1)
    lens = [(rng.randint(1, 9), rng.randint(1, 9)) for _ in range(9)]
    items = [(i, _utt(P, G, i + 1)) for i, (P, G) in enumerate(lens)]
    # every active row's table row is the reference rule at its utterance's (P, G, g_idx)
    m2 = FakeGPT()
    orig = m2.forward_step
    checked = []

    def fwd(cur, *, audio_valid, **kw):
        for r in range(m2.B):
            if m2.active[r]:
                i = (int(cur[r, 1, 0]) if m2.step[r] == 0 else int(m2.tag[r])) - 1
                P, G = lens[i]
                checked.append(i)
                assert audio_valid[r].tolist() == reference_rule(P, G, int(m2.step[r])), (i, int(m2.step[r]))
        return orig(cur, audio_valid=audio_valid, **kw)

    m2.forward_step = fwd
    done = dict(InferenceImp(None, m2, "sampling", 0.7, 25, 0.8, 30, "TTS").generate_many(items, capacity=3))
    assert sorted(done) == list(range(9))
    assert sorted(set(checked)) == list(range(9)) and len(checked) == sum(G for _, G in lens)


def test_capacity_is_bounded():
    import pytest
    from rstnet_b200._lib import RstnetError
    imp = InferenceImp(None, FakeGPT(), "sampling", 0.7, 25, 0.8, 30, "TTS")
    for cap in (0, 257):
        with pytest.raises(RstnetError):
            next(imp.generate_many([("a", _utt(2, 2, 1))], capacity=cap))


def test_new_abi_symbols_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    assert "int rstnet_counter_add_rows(" in header and "rstnet_counter_add_rows" in _lib.SYMBOLS
    # the row map is two arguments of the uniform entry points, straight after offset_stride
    for name in ("rstnet_lm_rope_kv_append_bf16", "rstnet_lm_ring_decode_attention_bf16"):
        decl = header[header.index(f"int {name}("):]
        decl = " ".join(re.sub(r"\s*/\*.*?\*/", "", decl[:decl.index(");")]).split())
        assert "int32_t offset_stride, const int32_t* row_stream, const int32_t* row_tl," in decl, (name, decl)
        assert name in _lib.SYMBOLS
    lib = _lib.lib()
    for name in ("rstnet_lm_rope_kv_append_rows_bf16", "rstnet_lm_ring_decode_attention_rows_bf16", "rstnet_lm_sample_rows_bf16",
                 "rstnet_lm_sample_bf16"):
        assert name not in header and name not in _lib.SYMBOLS, name
        assert not hasattr(lib, name), name
    assert lib.rstnet_version() == 206
    capi = open(os.path.join(ROOT, "rstnet_b200", "csrc", "capi.cu")).read()
    assert "rstnet_version(void) { return 206; }" in capi


@pytest.mark.parametrize("name", ["rstnet_lm_rope_kv_append_bf16", "rstnet_lm_ring_decode_attention_bf16"])
def test_row_map_arguments_are_checked(name):
    """Half a row map, or a row map with a shared offset (offset_stride 0), is an error return before any launch.  Every call
    also carries n_kv 0, which the entry points reject later, so none of them can reach a launch."""
    lib = _lib.lib()
    fake = 1 << 20      # non-NULL pointers that are never dereferenced
    fn = getattr(lib, name)

    def call(offset_stride, row_stream, row_tl):
        if name == "rstnet_lm_rope_kv_append_bf16":
            return fn(fake, fake, fake, 64, 64, fake, offset_stride, row_stream, row_tl, fake, fake, 5, 2, 4, 0, 64, 16, None)
        return fn(fake, fake, fake, offset_stride, row_stream, row_tl, fake, 5, 2, 4, 0, 64, 16, 16, None)

    for args, msg in (((1, fake, None), "row_stream and row_tl go together"), ((1, None, fake), "row_stream and row_tl go together"),
                      ((0, fake, fake), "a row map needs per-stream offsets")):
        assert call(*args) != 0, args
        assert msg in lib.rstnet_last_error().decode(), args
    # the map's own checks pass with both pointers and offset_stride 1 (and rows 5 need not be a multiple of B 2): n_kv 0 fails
    assert call(1, fake, fake) != 0
    assert "multiple of n_kv" in lib.rstnet_last_error().decode()
    assert call(1, None, None) != 0
    assert "multiple of the stream count" in lib.rstnet_last_error().decode()
