"""The reference loop's four tasks without a GPU: oracle/task_oracle.py against tests/golden/lm_tasks.npz (the unmodified
reference loop, read by oracle/gen_golden_tasks.py) and against today's TTS goldens, InferenceImp's layouts and
requests, the page reservation of a row that stops, and the ABI declaration of rstnet_lm_gen_rows_advance."""
import os

import numpy as np
import pytest
import torch

from oracle import gen_golden_tasks as GT
from oracle import infer_oracle as IO
from oracle import lm_oracle as L
from oracle import task_oracle as T
from rstnet_b200._lib import RstnetError
from rstnet_b200.infer import InferenceImp, candidate_counts, continuation_codes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "lm_tasks.npz"))


@pytest.mark.parametrize("mode,use_sampling", [("greedy", False), ("top1", True)])
def test_task_oracle_equals_the_reference_loop(gold, mode, use_sampling):
    """every item of every task (fp32): frames, stop and window as the reference produced them; fp32 near-ties
    (margin < 1e-3) may flip across BLAS builds, so frames are compared up to the first one"""
    from oracle.gen_golden import weights_digest
    w = GT.task_weights()
    assert weights_digest(w) == str(gold["weights_sha256"])
    outcomes = set()
    for name in [str(n) for n in gold["items"]]:
        seq = torch.from_numpy(gold[f"{name}_seq"])
        task = str(gold[f"{name}_task"])
        lens = tuple(int(v) for v in gold[f"{name}_lengths"]) or None
        with torch.no_grad():
            r = T.inference_imp(task, w, GT.CFG, seq, use_sampling, lengths=lens)
        ref = torch.from_numpy(gold[f"{name}_f32_{mode}_frames"])
        m = torch.from_numpy(gold[f"{name}_f32_{mode}_margins"]).flatten()
        first = int((m < 1e-3).nonzero()[0]) if bool((m < 1e-3).any()) else m.numel()
        n = min(first, ref.numel(), r["frames"].numel())
        assert torch.equal(r["frames"].flatten()[:n], ref.flatten()[:n]), name
        assert [r["P"], r["minlen"], r["maxlen"]] == gold[f"{name}_f32_{mode}_window"].tolist(), name
        if first == m.numel():
            assert torch.equal(r["frames"], ref) and r["stopped"] == bool(gold[f"{name}_f32_{mode}_stopped"]), name
        outcomes.add((task, bool(gold[f"{name}_f32_{mode}_stopped"])))
    # the fixture holds ASR items that stop inside their window and ASR items that run to maxlen
    assert ("ASR", True) in outcomes and ("ASR", False) in outcomes and ("TTS", True) in outcomes


def test_fixed_window_reduces_to_the_tts_oracle():
    """lengths = (G, G) on TTS is today's oracle bit for bit (and its goldens, lm_round2.npz)"""
    gold = np.load(os.path.join(ROOT, "tests", "golden", "lm_round2.npz"))
    cfg = L.SMALL
    w = L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05)
    seq = torch.from_numpy(gold["infer_seq"])
    G = int(seq[0].eq(T.TEXT_EMPTY).sum())
    for mode, use_sampling in (("greedy", False), ("top1", True)):
        with torch.no_grad():
            a = IO.inference_imp_tts(w, cfg, seq.clone(), use_sampling)
            b = T.inference_imp("TTS", w, cfg, seq.clone(), use_sampling, lengths=(G, G))
            c = T.inference_imp("TTS", w, cfg, seq.clone(), use_sampling)
        for r in (b, c):
            assert torch.equal(a["frames"], r["frames"]) and torch.equal(a["codes"], r["codes"])
            assert torch.equal(a["margins"], r["margins"]) and not r["stopped"]
        ref = torch.from_numpy(gold[f"infer_f32_{mode}_frames"])
        m = torch.from_numpy(gold[f"infer_f32_{mode}_margins"]).flatten()
        first = int((m < 1e-3).nonzero()[0]) if bool((m < 1e-3).any()) else m.numel()
        assert torch.equal(b["frames"].flatten()[:first], ref.flatten()[:first])


def test_layouts_of_every_task(gold):
    """InferenceImp._layout equals the oracle's restatement of infer_no_streaming.py:184-226 on every fixture item and
    on edge cases (pads of the other task's kind are not stripped; ASR's prompt is at most the sequence)"""
    imp = InferenceImp(None, None, "sampling", 0.7, 25, 0.8, 30, "TTS")
    for name in [str(n) for n in gold["items"]]:
        seq = torch.from_numpy(gold[f"{name}_seq"])
        task = str(gold[f"{name}_task"])
        _, P, lo, hi = T.layout(task, seq)
        assert imp._layout(seq, task) == (P, lo, hi), name
    asr = GT.task_sequence("ASR", 6, 14, 2, 41)
    assert imp._layout(asr, "ASR") == (7, 20 - 6 - 13, 20 - 6 + 13)
    assert imp._layout(asr, "text_only") == (10, 10, 10)          # two text-pad frames stripped: L = 20
    assert imp._layout(asr, "audio_only") == (3, 3, 3)            # row 1's 16 acoustic pads count as semantic: L = 6
    only_audio = torch.full((9, 5), 7)
    only_audio[0] = T.TEXT_EMPTY
    assert imp._layout(only_audio, "ASR") == (5, 5 - 5 - 13, 13) == T.layout("ASR", only_audio)[1:]
    with pytest.raises(RstnetError, match="2 frames"):
        imp._layout(torch.full((9, 1), 7), "audio_only")
    with pytest.raises(NotImplementedError):
        imp._layout(asr, "word_level_audio_text_alignment")
    with pytest.raises(RstnetError, match="nothing to generate"):
        imp._layout(torch.full((9, 4), 7), "TTS")


def test_requests_and_windows():
    imp = InferenceImp(None, None, "sampling", 0.7, 25, 0.8, 30, "TTS")
    tts = GT.task_sequence("TTS", 5, 8, 2, 11)
    # (utt, seq, P, G = maxlen, sampling, seed, task, minlen, windowed)
    assert imp._request("a", tts, None, 3)[2:] == (5, 8, None, 3, "TTS", 8, False)
    assert imp._request("a", tts, None, 3, lengths=(3, 20))[2:] == (5, 20, None, 3, "TTS", 3, True)
    assert imp._request("a", tts, None, 3, lengths=(19, 20))[8] is False     # maxlen - 1 <= minlen: never stops
    assert imp._request("a", tts, None, 3, lengths=(0, 1))[8] is False
    assert imp._request("a", tts, None, 3, lengths=(-1, 1))[8] is True       # frame 0 > minlen: it may stop
    assert imp._request("a", GT.task_sequence("audio_only", 7, 8, 0, 22), None, 0, "audio_only")[2:] == \
        (7, 7, None, 0, "audio_only", 7, False)
    asr = imp._request("a", GT.task_sequence("ASR", 6, 14, 2, 41), None, 0, "ASR")
    assert asr[2:] == (7, 27, None, 0, "ASR", 1, True)
    for bad in ((1,), (1, 0), (1.0, 5), (True, 5), (0, 2 ** 31), "ab"):
        with pytest.raises(RstnetError):
            imp._request("a", tts, None, 0, lengths=bad)
    for task in ("TTS", "audio_only", "text_only", "ASR"):
        InferenceImp(None, None, "sampling", 0.7, 25, 0.8, 30, task)._check_task()
    with pytest.raises(NotImplementedError):
        InferenceImp(None, None, "sampling", 0.7, 25, 0.8, 30, "dialogue")._check_task()
    # streaming runs the audio tasks, with or without an open window; the text tasks raise
    imp._check_streamed(imp._request("a", tts, None, 0, lengths=(3, 20)))
    imp._check_streamed(imp._request("a", GT.task_sequence("audio_only", 7, 8, 0, 22), None, 0, "audio_only"))
    imp._check_streamed(imp._request("a", tts, None, 0))
    for task in ("text_only", "ASR"):
        with pytest.raises(RstnetError, match="generates text"):
            imp._check_streamed(imp._request("a", GT.task_sequence(task, 6, 14, 2, 41), None, 0, task))
        with pytest.raises(NotImplementedError):
            InferenceImp(None, None, "sampling", 0.7, 25, 0.8, 30, task)._check_many(2, None, streamed=True)


def test_candidate_counts_with_any_minlen():
    """the host rule (candidate_counts) equals the oracle's branch restatement for negative, small and large minlen"""
    for P in (1, 5, 9):
        for minlen in (-14, -1, 0, 3, 8, 40):
            for g in range(0, 30):
                assert candidate_counts(P, minlen, g) == [T.n_valid(P, minlen, g, l) for l in range(8)], (P, minlen, g)


def test_continuation_codes():
    seq = GT.task_sequence("audio_only", 6, 4, 3, 5)         # L = 10 after its 3 pad frames: P = 5
    frames = torch.randint(0, 2048, (7, 9), generator=torch.Generator().manual_seed(2))
    codes = continuation_codes(seq, frames)
    whole = torch.cat([seq[1:, :5], frames[:, 1:].t()], 1)   # [8, 12]
    assert codes.shape == (8, 11)
    assert torch.equal(codes[0], whole[0, :-1]) and torch.equal(codes[1:], whole[1:, 1:])
    # at the join: the prompt's last frame takes codebooks 1..7 from the first generated frame
    assert torch.equal(codes[1:, 4], frames[0, 2:])
    assert torch.equal(continuation_codes(seq, frames[:0]), torch.cat([seq[1:2, :4], seq[2:, 1:5]], 0))


class _Pages:
    """stand-in allocator: counts reserved positions per row"""

    def __init__(self, n_pages, page):
        self.n_pages, self.page, self.free, self.held = n_pages, page, n_pages, {}

    def pages_for(self, n):
        return -(-n // self.page)

    def reserve(self, rows, n):
        for r in rows:
            self.held[r] = self.pages_for(n)
            self.free -= self.held[r]

    def release(self, rows):
        for r in rows:
            self.free += self.held.pop(r)


def test_pages_of_a_stopped_row_released_when_its_status_is_read():
    """a windowed row reserves P + maxlen positions and gives them all back when its stop is learned, one frame late;
    the frames it ran after the stop are dropped from its result"""
    from rstnet_b200 import _lib
    from rstnet_b200.infer import _Row, _TTSRows
    rows = _TTSRows.__new__(_TTSRows)
    rows.B, rows.dep_q, rows.dev, rows.paged = 2, 8, torch.device("cpu"), True
    rows.pages = _Pages(8, 16)
    rows.m = type("M", (), {"reset_streaming": lambda self, streams: None})()
    rows.dirty, rows.lp_frames = set(), {}
    imp = InferenceImp(None, None, "sampling", 0.7, 25, 0.8, 30, "TTS")
    req = imp._request("u", GT.task_sequence("ASR", 6, 14, 2, 41), None, 0, "ASR")
    P, G = req.P, req.G
    rows.pages.reserve([1], P + G)
    assert rows.pages.held[1] == rows.pages.pages_for(7 + 27)
    st = _Row("u", P, G, 3, None, "ASR", req.minlen, True, cand=0, group=0, g=4)
    rows.rows = [None, st]
    # frames 3..8 ran (the host has enqueued frame 8); the statuses of frame 7 say row 1 stopped there
    rows.history = {f: torch.full((2, 9), f, dtype=torch.int64) for f in range(3, 9)}
    rows.n = 9
    rows.status = [torch.tensor([_lib.GEN_IDLE, _lib.GEN_STOPPED], dtype=torch.int32), None]
    rows.lagged = (7, 0, None, {1: st}, None)
    done = rows.settle()
    assert rows.rows == [None, None] and rows.pages.free == 8 and 1 in rows.dirty
    (utt, codes, raw, fin), = done
    assert utt == "u" and codes is None and fin.frames == 4 and fin.stopped
    assert raw[:, 0].tolist() == [3, 4, 5, 6]      # frames 7 (stopped) and 8 (run after the stop) dropped
    assert not rows.history                        # nothing left to keep


def test_abi_declares_and_binds_gen_rows_advance():
    from rstnet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    assert "int rstnet_lm_gen_rows_advance(" in header and "rstnet_lm_gen_rows_advance" in _lib.SYMBOLS
    assert "#define RSTNET_GEN_REC 5" in header and _lib.GEN_REC == 5
    for name, v in (("HELD", 0), ("FIXED", 1), ("WINDOWED", 2), ("ARGMAX", 4), ("RUNNING", 0), ("LAST", 1), ("STOPPED", 2),
                    ("IDLE", 3)):
        assert f"RSTNET_GEN_{name} = {v}" in header and getattr(_lib, f"GEN_{name}") == v
    lib = _lib.lib()
    assert len(lib.rstnet_lm_gen_rows_advance.argtypes) == 10
    assert lib.rstnet_lm_gen_rows_advance(None, 9, None, None, 8, None, 4, 8, 2050, None) != 0   # refused before any launch
    assert b"null pointer" in lib.rstnet_last_error()
