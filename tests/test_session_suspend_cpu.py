"""Session suspend / resume, the parts that need no GPU: `FrameScheduler`'s suspend / resume bookkeeping over a stub engine
built on the engines' page policy (`serve._PagedRows`), the in-flight page accounting, `on_short="suspend"` on a churn
trace, the unchanged "evict" default, state compatibility, the segment tables of codec buffers, and the new entry points'
declarations."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from rstnet_b200 import _lib, row_state
from rstnet_b200._lib import RstnetError
from rstnet_b200.codec import _Buf
from rstnet_b200.lm import KVPages
from rstnet_b200.serve import FrameScheduler, _PagedRows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGE, CAP = 16, 40


class FakeEvent:
    def __init__(self):
        self.done = False

    def query(self):
        return self.done


class FakeLM:
    def __init__(self, n_pages, B):
        self._state = SimpleNamespace(pages=KVPages(n_pages, B, PAGE, CAP), pos_host=np.zeros(B, dtype=np.int64),
                                      upload_pages=lambda rows: None)

    def _paged(self):
        return self._state

    def reserve_kv(self, streams, positions):
        self._state.pages.reserve(streams, positions)

    def release_kv(self, streams):
        self._state.pages.release(streams)

    @property
    def kv_pages_free(self):
        return self._state.pages.free


class SwapStub(_PagedRows):
    """The host side of an engine with suspend_rows / resume_rows: a state is the row's position; a gather completes
    when the test says so (`finish`)."""

    def __init__(self, B, n_pages):
        self.B, self.kv_pages, self._kv_lm = B, n_pages, FakeLM(n_pages, B)
        self._in_flight, self.events, self.resumed = [], [], []

    def reset_rows(self, rows):
        self._reserve_first_page(rows)
        self._kv_lm._state.pos_host[list(rows)] = 0

    def step(self, pcm_rows, active):
        st = self._kv_lm._state
        st.pages.check(active, st.pos_host[active], 1)
        st.pos_host[active] += 1
        return {r: (f"tok{r}", pcm_rows[r]) for r in active}

    def suspend_rows(self, rows):
        out = []
        for r in rows:
            ev = FakeEvent()
            self.events.append(ev)
            self._in_flight.append((ev, self._kv_lm._state.pages.detach(r)))
            out.append(SimpleNamespace(positions=int(self._kv_lm._state.pos_host[r])))
        return out

    def resume_rows(self, rows, states):
        self.reclaim()
        self._kv_lm.reserve_kv(rows, [s.positions for s in states])
        for r, s in zip(rows, states):
            self._kv_lm._state.pos_host[r] = s.positions
            self.resumed.append((r, s.positions))

    def finish(self):
        for ev in self.events:
            ev.done = True


def _push_all(sch, t):
    for s in list(sch.sessions()) + sch.suspended():
        sch.push(s, f"{s}{t}")


def test_suspend_keeps_queue_and_in_flight_pages():
    eng = SwapStub(3, 6)
    sch = FrameScheduler(eng, 3)
    sch.admit("A")
    sch.admit("B")
    for t in range(20):                                        # A and B cross position 16: two pages each
        _push_all(sch, t)
        sch.tick()
    assert eng.kv_pages_free == 2
    sch.suspend("A")
    assert sch.suspended() == ["A"] and sch.sessions() == {"B": 1} and sch.free_rows() == 2
    assert eng.kv_pages_free == 2                              # A's pages are in flight: not free yet
    assert eng.reclaim() == 0 and eng.kv_pages_free == 2
    sch.push("A", "a-late")                                    # a suspended session keeps queueing
    assert len(sch._queue["A"]) == 1
    eng.finish()
    assert eng.reclaim() == 2 and eng.kv_pages_free == 4
    assert sch.resume("A") == 0                                # the lowest free row
    assert sch.sessions() == {"B": 1, "A": 0} and sch.suspended() == []
    assert eng.resumed == [(0, 20)] and eng._kv_lm._state.pages.held[0] == 2
    out = sch.tick()
    assert out["A"] == ("tok0", "a-late")
    assert sch.suspensions == 1 and sch.resumes == 1 and sch.lag == {"A": 0}


def test_next_tick_returns_in_flight_pages():
    eng = SwapStub(2, 3)
    sch = FrameScheduler(eng, 2)
    sch.admit("A")
    sch.admit("B")
    sch.suspend("A")
    assert eng.kv_pages_free == 1
    eng.finish()
    _push_all(sch, 0)
    sch.tick()                                                 # grow_kv reclaims first
    assert eng.kv_pages_free == 2


def test_resume_order_and_release_of_a_suspended_session():
    eng = SwapStub(4, 12)
    sch = FrameScheduler(eng, 4)
    for s in "ABCD":
        sch.admit(s)
    for s in ("C", "A", "D"):
        sch.suspend(s)
    assert sch.suspended() == ["C", "A", "D"]
    sch.release("A")                                           # a suspended session can end: its state is dropped
    assert sch.suspended() == ["C", "D"]
    with pytest.raises(KeyError):
        sch.push("A", "x")
    eng.finish()
    assert sch.resume("D") == 0 and sch.resume("C") == 2
    with pytest.raises(RuntimeError):
        sch.resume("C")


def _churn(on_short, n_pages=10, ticks=140, B=6):
    """sessions arrive every 9 ticks and run 60 ticks; a pool of n_pages pages of 16 cannot hold them all"""
    eng = SwapStub(B, n_pages)
    sch = FrameScheduler(eng, B, on_short=on_short)
    evicted, steps, ended, arrive = [], {}, [], {}
    for t in range(ticks):
        eng.finish()                                           # each tick's gathers have completed by the next
        if t % 9 == 0 and sch.free_rows() and eng.kv_pages_free >= 1:
            s = f"s{t}"
            sch.admit(s)
            arrive[s] = t
        for s in list(sch.sessions()) + sch.suspended():
            if t - arrive[s] < 60:
                sch.push(s, t)
        for s in sch.tick():
            steps[s] = steps.get(s, 0) + 1
        evicted += sch.take_evicted()
        for s in list(sch.sessions()):
            if steps.get(s, 0) >= 60:
                sch.release(s)
                ended.append(s)
    return sch, evicted, steps, ended


def test_on_short_suspend_evicts_nobody():
    sch, evicted, steps, ended = _churn("evict")
    assert evicted                                             # the trace is short of pages
    sch, evicted, steps, ended = _churn("suspend")
    assert evicted == [] and sch.suspensions > 0 and sch.resumes > 0
    assert all(steps[s] == 60 for s in ended) and len(ended) >= 5
    assert max(sch.lag.values()) > 0


def test_evict_default_unchanged():
    """the default scheduler makes no suspend / resume call, and evicts as before"""
    eng = SwapStub(4, 5)
    sch = FrameScheduler(eng, 4)
    assert sch.on_short == "evict"
    for s in ("C", "A", "B"):
        sch.admit(s)
    for t in range(16):
        _push_all(sch, t)
        sch.tick()
    _push_all(sch, 16)
    assert set(sch.tick()) == {"C", "A"} and sch.take_evicted() == ["B"]
    assert eng.events == [] and sch.suspended() == [] and eng.kv_pages_free == 1
    with pytest.raises(RstnetError):
        FrameScheduler(eng, 4, on_short="drop")


def test_incompatible_state_raises():
    blob = torch.zeros(16, dtype=torch.uint8)
    regions = [("kv", row_state.segs((4096, 64, 64, 2)))]
    st = row_state.SessionState(("DuplexEngine", "cfg", (1,), 24000, 64), row_state.signature(regions), blob, 128, {"pos": 3})
    row_state.check_compatible(st, st.key, regions)
    for key in (("MoshiDuplexEngine", "cfg", (1,), 24000, 64), ("DuplexEngine", "cfg", (1,), 16000, 64),
                ("DuplexEngine", "cfg", (1,), 24000, 32), ("DuplexEngine", "other", (1,), 24000, 64)):
        with pytest.raises(RstnetError):
            row_state.check_compatible(st, key, regions)
    with pytest.raises(RstnetError):
        row_state.check_compatible(st, st.key, [("kv", row_state.segs((4096, 64, 64, 3)))])
    with pytest.raises(RstnetError):
        row_state.check_compatible("not a state", st.key, regions)
    assert st.positions == 3


@pytest.mark.parametrize("tbc", [True, False])
def test_buf_segments(tbc):
    B, ctx, T, extra, C = 5, 3, 4, 1, 6
    buf = _Buf(B, ctx, T, extra, C, "cpu", tbc)
    base, rows = buf.t.data_ptr(), ctx + T + extra
    for b in (0, 2, 4):
        s = buf.row_segments(b)
        if tbc:                          # [rows, B, C]: ctx pieces of C floats, one time step apart
            assert s.tolist() == [[base + 4 * b * C, 4 * B * C, 4 * C, ctx]]
        else:                            # [B, rows, C]: the ctx rows are one contiguous piece
            assert s.tolist() == [[base + 4 * b * rows * C, 4 * ctx * C, 4 * ctx * C, 1]]
        # the bytes the segments name are exactly the carry rows of stream b, in row order
        flat = buf.t.view(-1)
        buf.t.copy_(torch.randn_like(buf.t))
        picked = torch.cat([flat[(a - base) // 4 + k * st // 4:(a - base) // 4 + k * st // 4 + n // 4]
                            for a, st, n, cnt in s.tolist() for k in range(cnt)])
        want = buf.t[:ctx, b] if tbc else buf.t[b, :ctx]
        assert torch.equal(picked, want.reshape(-1))
    assert len(_Buf(B, 0, T, 0, C, "cpu", tbc).row_segments(1)) == 0


def test_layout_aligns_regions():
    regions = [("a", row_state.segs((1000, 7, 7, 3))), ("b", row_state.segs()), ("c", row_state.segs((2000, 8, 8, 1), (3000, 8, 8, 2)))]
    table, n = row_state.layout(regions)
    assert table["staging_offset"].tolist() == [0, 32, 40] and n == 64
    assert table["count"].tolist() == [3, 1, 2] and table.itemsize == 40


def test_segment_symbols_in_header_and_lib():
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    assert "rstnet_segment;" in header
    for name in ("rstnet_segments_gather", "rstnet_segments_scatter"):
        assert f"int {name}(" in header and name in _lib.SYMBOLS
        assert getattr(_lib.lib(), name).argtypes
