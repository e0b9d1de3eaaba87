"""Equivalence test of the batch TTS loop (`infer._TTSRows`) behind generate_many, stream_many and serve.TTSEngine.

A recording stand-in model runs the loop on the CPU: a real lm.KVPages for the pages, the gen_rows stop rule of
gen_rows.cu, per-row log-probability sums, prompt forks and a codec with its delay cache.  Every call the loop makes to
it, with its arguments, and every value the loop yields are logged, over a seeded mixed corpus: fixed TTS, TTS with open
windows, audio_only, ASR and text_only items with per-row sampling and short page pools, best-of-N with fixed and windowed
candidates, and streamed generation with windowed rows that stop.  The log is compared with tests/golden/tts_rows_log.npz,
so any change to admissions, page use, launches, copies, completion order or results shows up here.

    python tests/test_tts_rows_cpu.py --record      # rewrite the golden log from the current loop
"""
import json
import os
import sys
from contextlib import contextmanager

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import gen_golden_tasks as GT  # noqa: E402
from rstnet_b200 import _lib, infer  # noqa: E402
from rstnet_b200.infer import InferenceImp, Sampling  # noqa: E402
from rstnet_b200.lm import KVPages  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "tts_rows_log.npz")
PAGE, CONTEXT, FS = 16, 32, 1920


def plain(x):
    """a JSON-able form of a logged value"""
    if isinstance(x, torch.Tensor):
        return plain(x.tolist())
    if isinstance(x, np.ndarray):
        return plain(x.tolist())
    if isinstance(x, (np.integer, np.floating, np.bool_)):
        return x.item()
    if isinstance(x, Sampling):
        return repr(x)
    if isinstance(x, infer.TTSChunk):
        pcm = x.pcm
        return ["chunk", plain(x.utt_id), x.index, pcm.numel(), plain(pcm[:10]), float(pcm.double().sum()), plain(x.codes)]
    if isinstance(x, dict):
        return [[plain(k), plain(v)] for k, v in sorted(x.items(), key=lambda kv: repr(kv[0]))]
    if isinstance(x, (list, tuple)):
        return [plain(v) for v in x]
    return x


def _mix(*vals) -> int:
    h = 0x345678
    for v in vals:
        h = ((h ^ (int(v) & 0xFFFFFFFFFFFF)) * 0x100000001B3 + 0x9E3779B9) & 0xFFFFFFFFFFFFFFFF
        h ^= h >> 29
    return h & 0x3FFFFFFFFFFFFFFF


class FakeState:
    """the LM scope's host and device state the loop reads: pages, page uploads, generation records and statuses,
    log-probability sums"""

    def __init__(self, m, B, kv_pages):
        self.m, self.B = m, B
        self.pages = KVPages(kv_pages, B, PAGE, CONTEXT)
        self.pos = np.zeros(B, dtype=np.int64)
        self.gen_rec = np.zeros((B, _lib.GEN_REC), dtype=np.int64)
        self.row_valid = np.full((B, 8), 2048, dtype=np.int64)
        self.gen_status = torch.full((B,), _lib.GEN_IDLE, dtype=torch.int32)
        self.lp_acc = None
        self.active = np.zeros(B, dtype=np.int64)

    def upload_pages(self, streams):
        self.m.rec("upload_pages", list(streams), self.pages.table[list(streams)])

    def gen_rows_set(self, rows, records, valid):
        self.m.rec("gen_rows_set", rows, records, valid)
        self.gen_rec[list(rows)] = np.asarray(records)
        self.row_valid[list(rows)] = np.asarray(valid)

    def logprob_reset(self, rows=None):
        self.m.rec("logprob_reset", rows)
        if self.lp_acc is None:
            self.lp_acc = torch.zeros(self.B, 9, dtype=torch.float64)
        elif rows is None:
            self.lp_acc.zero_()
        else:
            self.lp_acc[list(rows)] = 0

    def logprob_sums(self):
        self.m.rec("logprob_sums")
        return self.lp_acc.clone()

    def write(self, rows, n, cow_rows):
        """what _LMState does before a launch in which `rows` write n positions and `cow_rows` their next n slots: the
        page check and copy-on-write"""
        self.pages.check(rows, self.pos[rows], n)
        pairs, changed = self.pages.cow(cow_rows, self.pos[cow_rows], n)
        if pairs:
            self.m.rec("cow", pairs, changed)
        self.pos[rows] += n


class FakeGPT:
    """GPT's streaming protocol for the batch loop.  A row's tokens at its generated frame g are a hash of its prompt (kept
    through a fork), its random-stream key, its sampling settings and g; an audio codebook whose candidate set includes
    id 2048 takes it about once in 40 frames, so windowed rows stop.  The generation records advance as gen_rows.cu does."""
    num_codebooks = 9
    device = torch.device("cpu")

    class config:
        context = CONTEXT
        audio_card = 2050

    def __init__(self, log):
        self.log = log
        self._state = None

    def rec(self, *entry):
        self.log.append(plain(entry))

    @contextmanager
    def streaming(self, B, kv_pages=None):
        self.rec("streaming", B, kv_pages)
        self._state = FakeState(self, B, kv_pages)
        self.B = B
        self.step = np.zeros(B, dtype=np.int64)
        self.tag = np.zeros(B, dtype=np.int64)
        self.keys = np.zeros(B, dtype=np.int64)
        try:
            yield
        finally:
            self._state = None
            self.rec("exit")

    def reserve_kv(self, streams, positions):
        raise AssertionError("the loop reserves through the scope's allocator")

    def _get_initial_token(self):
        tok = torch.full([1, 9, 1], 2048, dtype=torch.long)
        tok[:, 0] = 151655
        return tok

    def set_active_streams(self, mask):
        self.rec("active", mask)
        self._state.active = np.asarray(mask, dtype=np.int64).copy()

    def reset_streaming(self, streams=None):
        self.rec("reset", streams)
        self._state.pos[list(streams)] = 0
        self.step[list(streams)] = 0

    def prefill_streams(self, prompts):
        self.rec("prefill", {r: [list(p.shape), int(p.sum())] for r, p in prompts.items()})
        for r, p in prompts.items():
            self._state.write([r], p.shape[1], [r])
            self.tag[r] = _mix(*p.reshape(-1).tolist())
            self.step[r] = 0

    def fork_kv(self, src, dsts, positions):
        st = self._state
        pairs, rows = st.pages.share(src, dsts, positions, int(st.pos[src]))
        self.rec("fork_kv", src, dsts, positions, pairs, st.pages.table[list(rows)])
        st.pos[list(rows)] = st.pos[src]
        self.tag[list(rows)] = self.tag[src]
        self.step[list(rows)] = self.step[src]

    def forward_step(self, cur, *, audio_valid=None, sample_key=None, sampling=None, gen_rows=False, logprob=False, **kw):
        st, B = self._state, self.B
        self.rec("step", cur[:, :, 0], audio_valid, sample_key, sampling, gen_rows, logprob, kw, st.active)
        if sample_key is not None:
            self.keys = np.asarray(sample_key, dtype=np.int64).copy()
        act = [r for r in range(B) if st.active[r]]
        st.write(act, 1, list(range(B)))     # held rows write their next slot too
        if logprob and st.lp_acc is None:
            st.logprob_reset()
        toks = torch.zeros(B, 9, dtype=torch.int64)
        for r in range(B):
            valid = st.row_valid[r] if gen_rows else (audio_valid[r] if audio_valid is not None else [2048] * 8)
            h = _mix(self.tag[r], self.keys[r], self.step[r], _mix(*map(ord, repr(sampling[r]))) if sampling else 0)
            toks[r, 0] = h % 128000
            for l in range(8):
                hl = _mix(h, l)
                toks[r, l + 1] = 2048 if int(valid[l]) > 2048 and hl % 40 == 0 else (hl >> 8) % 2048
        for r in act:
            self.step[r] += 1
            if st.lp_acc is not None and logprob:
                st.lp_acc[r] += torch.tensor([-((int(t) % 13) + 1) / 8.0 for t in toks[r]], dtype=torch.float64)
        if gen_rows:
            self._advance(toks)
        return toks

    def _advance(self, toks):
        """gen_rows.cu's rstnet_lm_gen_rows_advance on every row"""
        st = self._state
        for b in range(self.B):
            pre, minlen, maxlen, g, mode = (int(v) for v in st.gen_rec[b])
            kind = mode & 3
            if kind not in (_lib.GEN_FIXED, _lib.GEN_WINDOWED):
                st.gen_status[b] = _lib.GEN_IDLE
                continue
            stop = kind == _lib.GEN_WINDOWED and g > minlen and any(int(toks[b, 1 + l]) >= 2048 for l in range(3, 8))
            if stop or g + 1 >= maxlen:
                st.gen_status[b] = _lib.GEN_STOPPED if stop else _lib.GEN_LAST
                st.gen_rec[b, 4] = mode & ~3
                continue
            st.gen_rec[b, 3] = g + 1
            st.gen_status[b] = _lib.GEN_RUNNING
            argmax = mode & _lib.GEN_ARGMAX
            st.row_valid[b] = [self.config.audio_card if argmax else (2049 if l > 0 and pre + g + 1 > minlen else 2048)
                               for l in range(8)]

    def check_device_errors(self):
        self.rec("check")


class FakeDelay:
    """the TTS delay of rstnet_lm_delay_cache_out restated: after a row's generated frame f >= 1, out[1:] is codebook 0 of
    frame f - 1 and codebooks 1-7 of frame f; held rows keep their state"""

    def __init__(self, m, B):
        self.m, self.B = m, B
        self.prev = torch.zeros(B, 9, dtype=torch.long)
        self.off = np.zeros(B, dtype=np.int64)
        self.out = torch.zeros(B, 9, dtype=torch.long)
        self.valid = torch.zeros(B, dtype=torch.long)

    def reset(self, rows):
        self.m.rec("delay_reset", rows)
        for r in rows:
            self.off[r] = 0
            self.valid[r] = 0

    def step(self, toks):
        for b in range(self.B):
            if self.m._state.active[b]:
                self.out[b, :2] = self.prev[b, :2]
                self.out[b, 2:] = toks[b, 2:]
                self.prev[b] = toks[b]
                self.off[b] += 1
                self.valid[b] = int(self.off[b] > 1)
        return self.out, self.valid


class FakeCodec:
    """decode: pcm[b, :8] = row b's codes, pcm[b, 8] = the decode calls so far, pcm[b, 9] = the row's advance flag"""
    codebook_size = 2048
    frame_size = FS

    def __init__(self, m):
        self.m, self.calls = m, 0

    @contextmanager
    def streaming(self, B, clip_window=False):
        self.m.rec("codec_streaming", B, clip_window)
        self.B = B
        self.mask = torch.zeros(B, dtype=torch.long)
        yield
        self.m.rec("codec_exit")

    def reset_streaming(self, streams=None):
        self.m.rec("codec_reset", streams)

    def set_active_streams(self, mask):
        self.m.rec("codec_active", mask)
        self.mask = torch.as_tensor(mask).clone()

    def decode(self, codes):
        self.calls += 1
        self.m.rec("decode", codes[:, :, 0])
        pcm = torch.zeros(self.B, 1, FS)
        pcm[:, 0, :8] = codes[:, :, 0].float()
        pcm[:, 0, 8] = self.calls
        pcm[:, 0, 9] = self.mask.float()
        return pcm


def fake_event(log):
    """a torch.cuda.Event stand-in that logs its records and synchronises"""
    count = [0]

    class Event:
        def __init__(self, *a, **k):
            self.id = count[0]
            count[0] += 1

        def record(self, *a):
            log.append(["event_record", self.id])

        def synchronize(self):
            log.append(["event_sync", self.id])

        def query(self):
            return True
    return Event


# ---------------------------------------------------------------------------------------------------------------- corpus
def _corpus(seed):
    """a seeded mix of items -> (items, tasks, lengths, sampling, seeds)"""
    g = np.random.default_rng(seed)
    items, tasks, lengths, sampling, seeds = [], {}, {}, {}, {}
    kinds = ["TTS", "TTS_open", "audio_only", "ASR", "text_only"]
    for i in range(14):
        kind = kinds[int(g.integers(len(kinds)))] if i >= len(kinds) else kinds[i]
        task = "TTS" if kind == "TTS_open" else kind
        a, b = int(g.integers(2, 7)), int(g.integers(1, 9))
        u = f"u{i}"
        items.append((u, GT.task_sequence(task, a, b, int(g.integers(0, 3)), seed * 100 + i)))
        tasks[u] = task
        if kind == "TTS_open":
            lengths[u] = (int(g.integers(0, 3)), int(g.integers(4, 14)))
        seeds[u] = int(g.integers(0, 2 ** 31))
        if i % 4 == 1:
            sampling[u] = Sampling(True, 0.5, 5, 0.0, 0.9, 7, 0.0)
        elif i % 4 == 3:
            sampling[u] = Sampling(False)
    # prompts of more than one page, run past the ring (a forked candidate copies the shared page it wraps onto)
    for u, a, b, win in (("long0", 18, 20, None), ("long1", 17, 22, (1, 21))):
        items.append((u, GT.task_sequence("TTS", a, b, 1, seed * 100 + a)))
        tasks[u], seeds[u] = "TTS", seed + a
        if win is not None:
            lengths[u] = win
    return items, tasks, lengths, sampling, seeds


def _audio_corpus(seed):
    """audio items only, every other one with an open window"""
    g = np.random.default_rng(seed)
    items, tasks, lengths = [], {}, {}
    for i in range(9):
        task = "TTS" if i % 3 != 2 else "audio_only"
        a, b = int(g.integers(2, 6)), int(g.integers(1, 9))
        u = f"s{i}"
        items.append((u, GT.task_sequence(task, a, b, int(g.integers(0, 2)), seed * 100 + i)))
        tasks[u] = task
        if i % 2:
            lengths[u] = (int(g.integers(0, 3)), int(g.integers(5, 14)))
    return items, tasks, lengths


def _imp(m, task="TTS"):
    return InferenceImp(None, m, "sampling", 0.7, 25, 0.8, 30, task)


def _generate(log, cap, kv_pages, n_samples=1, return_frames=False, per_row=True, seed=1):
    m = FakeGPT(log)
    items, tasks, lengths, sampling, seeds = _corpus(seed)
    if n_samples > 1:      # best-of-N ranks candidates of the audio tasks and the text tasks alike
        items = items[:6] + items[-2:]
    stats = {}
    out = _imp(m).generate_many(items, cap, seeds=seeds, sampling=sampling if per_row else None, kv_pages=kv_pages,
                                stats=stats, n_samples=n_samples, tasks=tasks, lengths=lengths, return_frames=return_frames)
    for got in out:
        m.rec("yield", got)
    m.rec("stats", stats)


def _stream(log, cap, kv_pages):
    m = FakeGPT(log)
    items, tasks, lengths = _audio_corpus(3)
    for c in _imp(m).stream_many(items, cap, FakeCodec(m), seeds={u: i for i, (u, _) in enumerate(items)},
                                 sampling={items[1][0]: Sampling(True, 0.5, 5, 0.0, 0.9, 7, 0.0)}, kv_pages=kv_pages,
                                 tasks=tasks, lengths=lengths):
        m.rec("yield", c)


def _engine(log, cap, kv_pages):
    from rstnet_b200.serve import TTSEngine
    m = FakeGPT(log)
    items, tasks, lengths = _audio_corpus(4)
    with TTSEngine(_imp(m), FakeCodec(m), cap, kv_pages=kv_pages) as eng:
        for t in range(200):
            if t % 2 == 0 and items:
                u, s = items.pop(0)
                eng.submit(u, s, Sampling(False) if t % 6 == 4 else None, t, task=tasks[u], lengths=lengths.get(u))
            m.rec("engine_step", eng.step(), eng.pending, eng.active)
            if not items and not eng.pending and not eng.active:
                break


SCENARIOS = {
    "many_cap2_short": lambda log: _generate(log, 2, 3),
    "many_cap3_short": lambda log: _generate(log, 3, 4, seed=2),
    "many_cap3_frames": lambda log: _generate(log, 3, 12, return_frames=True, per_row=False),
    "best_of_3_cap3": lambda log: _generate(log, 3, 12, n_samples=3),
    "best_of_3_cap6_short": lambda log: _generate(log, 6, 8, n_samples=3, seed=2),
    "stream_cap2": lambda log: _stream(log, 2, 6),
    "stream_cap3_short": lambda log: _stream(log, 3, 3),
    "engine_cap3": lambda log: _engine(log, 3, 8),
}


def run_scenario(name, monkeypatch):
    log = []
    monkeypatch.setattr(infer, "_TTSDelay", FakeDelay)
    monkeypatch.setattr(torch.cuda, "Event", fake_event(log))
    SCENARIOS[name](log)
    return log


def _without_events(log):
    """the log without the event entries: on a CPU device the loop records no event (the parent of this test recorded
    one for the best-of-N sums that finishing rows copy, which a CPU device has nothing to wait for)"""
    return [e for e in log if e[0] not in ("event_record", "event_sync")]


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_loop_log_equals_golden(name, monkeypatch):
    log = run_scenario(name, monkeypatch)
    recorded = set()
    for e in log:       # an event is waited for only after it was recorded
        if e[0] == "event_record":
            recorded.add(e[1])
        elif e[0] == "event_sync":
            assert e[1] in recorded, e
    want = json.loads(bytes(np.load(GOLDEN)[name]).decode())
    got = json.loads(json.dumps(log))
    got, want = _without_events(got), _without_events(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a == b, f"{name}: entry {i} differs:\n got  {a}\n want {b}"
    assert len(got) == len(want), f"{name}: {len(got)} entries, {len(want)} in the golden log"


def test_corpus_reaches_every_path(monkeypatch):
    """the scenarios run what they are meant to: rows that stop and rows that run out, forks, page waits, chunks of
    stopped rows"""
    log = run_scenario("many_cap2_short", monkeypatch)
    stats = [e for e in log if e[0] == "stats"][0][1]
    assert dict(stats)["wait_frames"] > 0
    steps = [e for e in log if e[0] == "step"]
    assert any(e[5] for e in steps) and any(not e[5] for e in steps)          # frames with and without gen_rows
    assert any(e[0] == "gen_rows_set" and any(rec[4] & _lib.GEN_ARGMAX for rec in e[2]) for e in log)
    log = run_scenario("best_of_3_cap3", monkeypatch)
    assert any(e[0] == "fork_kv" for e in log) and any(e[0] == "cow" for e in log)
    cands = [c for e in log if e[0] == "yield" for c in e[1][1]]
    assert len({c[4] for c in cands}) > 2                                    # candidates of different lengths
    log = run_scenario("stream_cap2", monkeypatch)
    chunks = [e[1] for e in log if e[0] == "yield"]
    assert any(c[3] == 0 and c[6] is not None and c[2] > 0 for c in chunks)    # an empty last chunk: a row that stopped


def record():
    class MP:
        def __init__(self):
            self.undo = []

        def setattr(self, obj, name, value):
            self.undo.append((obj, name, getattr(obj, name)))
            setattr(obj, name, value)

        def close(self):
            for obj, name, value in reversed(self.undo):
                setattr(obj, name, value)
    out = {}
    for name in sorted(SCENARIOS):
        mp = MP()
        try:
            log = run_scenario(name, mp)
        finally:
            mp.close()
        out[name] = np.frombuffer(json.dumps(log).encode(), dtype=np.uint8)
        print(f"{name}: {len(log)} entries")
    np.savez_compressed(GOLDEN, **out)


if __name__ == "__main__":
    if "--record" in sys.argv[1:]:
        record()
