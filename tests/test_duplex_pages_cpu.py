"""Paged KV for duplex serving, the parts that need no GPU: `FrameScheduler`'s admission, growth and eviction policy over
a stub engine built on the engines' shared page policy (`serve._PagedRows`) and the host page allocator, and the new
paged pair-RoPE entry point's declaration and argument checks."""
import os
from types import SimpleNamespace

import numpy as np
import pytest

from rstnet_b200 import _lib
from rstnet_b200._lib import RstnetError
from rstnet_b200.lm import KVPages
from rstnet_b200.serve import FrameScheduler, _PagedRows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PAGE, CAP = 16, 40          # 3 pages per ring, the last one half used


class FakeLM:
    """The host side of a paged LM scope: the allocator, the position mirror, and the guard of a step."""

    def __init__(self, n_pages, B):
        self._state = SimpleNamespace(pages=KVPages(n_pages, B, PAGE, CAP), pos_host=np.zeros(B, dtype=np.int64))
        self.reserves = []

    def _paged(self):
        return self._state

    def reserve_kv(self, streams, positions):
        self.reserves.append((list(streams), positions))
        self._state.pages.reserve(streams, positions)

    def release_kv(self, streams):
        self._state.pages.release(streams)

    @property
    def kv_pages_free(self):
        return self._state.pages.free


class PagedStub(_PagedRows):
    def __init__(self, B, n_pages):
        self.B, self.kv_pages, self._kv_lm = B, n_pages, FakeLM(n_pages, B)
        self.resets, self.steps = [], []

    def reset_rows(self, rows):
        self._reserve_first_page(rows)
        self._kv_lm._state.pos_host[list(rows)] = 0
        self.resets.append(list(rows))

    def step(self, pcm_rows, active):
        st = self._kv_lm._state
        st.pages.check(active, st.pos_host[active], 1)         # the LM scope's guard: raises past a row's pages
        st.pos_host[active] += 1
        self.steps.append(list(active))
        return {r: (f"tok{r}", pcm_rows[r]) for r in active}


def _run(sch, sessions, ticks, gaps=()):
    """push one frame per tick for every live session (except (tick, session) in gaps) and tick"""
    evicted = {}
    for t in range(ticks):
        for s in sch.sessions():
            if (t, s) not in gaps:
                sch.push(s, f"{s}{t}")
        sch.tick()
        ev = sch.take_evicted()
        if ev:
            evicted[t] = ev
    return evicted


def test_admission_takes_a_page_and_release_returns_them():
    eng = PagedStub(3, 7)
    sch = FrameScheduler(eng, 3)
    assert sch.paged
    assert sch.admit("A") == 0 and eng.kv_pages_free == 6
    assert eng._kv_lm._state.pages.table[0].tolist() == [0, -1, -1]
    _run(sch, ["A"], 20)                                        # A crosses position 16: a second page
    assert eng._kv_lm._state.pages.held[0] == 2 and eng.kv_pages_free == 5
    sch.release("A")
    assert eng.kv_pages_free == 7
    _run(sch, [], 50)                                          # no session: nothing grows
    assert eng.kv_pages_free == 7


def test_growth_in_admission_order_and_eviction():
    """Pool of 5: A, B, C admitted (3 pages).  At position 16 all three want a second page at the same tick; the two
    oldest get one, the youngest is evicted, its row and pages returned, its frames dropped, and it is not stepped."""
    eng = PagedStub(4, 5)
    sch = FrameScheduler(eng, 4)
    for s in ("C", "A", "B"):                                  # admission order C, A, B (rows 0, 1, 2)
        sch.admit(s)
    ev = _run(sch, None, 16)
    assert ev == {} and eng.kv_pages_free == 2
    for s in ("C", "A", "B"):
        sch.push(s, "x")
    sch.push("B", "y")                                         # a second frame queued for B: dropped with B
    n = len(eng.steps)
    out = sch.tick()
    assert set(out) == {"C", "A"} and eng.steps[n] == [0, 1]
    assert sch.take_evicted() == ["B"] and sch.take_evicted() == []
    assert sch.sessions() == {"C": 0, "A": 1} and sch.free_rows() == 2 and eng.kv_pages_free == 1
    pages = eng._kv_lm._state.pages
    assert pages.held.tolist() == [2, 2, 0, 0]
    assert pages.table[0].tolist()[:2] == [0, 3] and pages.table[1].tolist()[:2] == [1, 4]   # oldest first, lowest page first
    with pytest.raises(KeyError):
        sch.push("B", "z")


def test_kv_headroom_refuses_and_changes_nothing():
    eng = PagedStub(4, 3)
    sch = FrameScheduler(eng, 4, kv_headroom=1)
    sch.admit("A")
    sch.admit("B")                                             # 1 free after: the headroom
    snap = (eng._kv_lm._state.pages.table.copy(), eng.kv_pages_free, sch.sessions(), sch.free_rows(), list(eng.resets))
    with pytest.raises(RuntimeError):
        sch.admit("C")
    assert np.array_equal(eng._kv_lm._state.pages.table, snap[0]) and eng.kv_pages_free == snap[1]
    assert sch.sessions() == snap[2] and sch.free_rows() == snap[3] and eng.resets == snap[4]
    assert FrameScheduler(PagedStub(1, 1), 1).admit("A") == 0   # default headroom 0: the last page is admissible
    with pytest.raises(RstnetError):
        FrameScheduler(eng, 4, kv_headroom=-1)


def test_held_session_does_not_grow():
    eng = PagedStub(2, 6)
    sch = FrameScheduler(eng, 2)
    sch.admit("A")
    sch.admit("B")
    gaps = {(t, "B") for t in range(10, 40)}                   # B sends nothing from tick 10 on
    _run(sch, None, 40, gaps)
    st = eng._kv_lm._state
    assert st.pos_host.tolist() == [40, 10]
    assert st.pages.held.tolist() == [3, 1]                    # A holds its whole ring, B still its first page
    assert all(1 not in rows for rows in eng.steps[10:])


def test_whole_ring_needs_no_more_pages():
    eng = PagedStub(1, 3)
    sch = FrameScheduler(eng, 1)
    sch.admit("A")
    assert _run(sch, None, 200) == {}
    assert eng._kv_lm._state.pages.held[0] == 3 and eng.kv_pages_free == 0
    assert len(eng._kv_lm.reserves) == 3                       # the first page, then one per boundary: 16 and 32


def test_grow_kv_returns_short_rows_unchanged():
    eng = PagedStub(3, 4)
    for r in range(3):
        eng.reset_rows([r])
    eng._kv_lm._state.pos_host[:] = [16, 5, 16]
    assert eng.grow_kv([2, 1, 0]) == [0]                       # row 2 first takes the last page; row 1 needs none
    pages = eng._kv_lm._state.pages
    assert pages.held.tolist() == [1, 1, 2] and pages.free == 0
    eng.release_rows([0, 1, 2])
    assert eng.kv_pages_free == 4


def test_plain_engine_sees_no_change():
    """An engine without kv_pages: no page calls, the same admissions, steps and results as before."""

    class Stub:
        def __init__(self):
            self.resets, self.steps = [], 0

        def reset_rows(self, rows):
            self.resets.append(list(rows))

        def step(self, pcm_rows, active):
            self.steps += 1
            return {r: (f"tok{r}", f"pcm{r}") for r in active}

    eng = Stub()
    s = FrameScheduler(eng, capacity=2, kv_headroom=5)
    assert not s.paged
    assert (s.admit("A"), s.admit("B")) == (0, 1)
    s.push("A", "a0")
    assert s.tick() == {"A": ("tok0", "pcm0")} and s.take_evicted() == []
    s.release("A")
    assert s.admit("C") == 0 and eng.resets == [[0], [1], [0]] and eng.steps == 1


def test_pair_append_paged_symbol_and_checks():
    name = "rstnet_lm_rope_pair_kv_append_paged_bf16"
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    assert f"int {name}(" in header and name in _lib.SYMBOLS
    lib = _lib.lib()
    assert getattr(lib, name).argtypes
    fake = 256                                                 # a pointer the checks never dereference
    for pt, stride, log2 in ((None, 13, 4), (fake, 13, 3), (fake, 13, 13), (fake, 12, 4), (fake, 0, 4)):
        assert getattr(lib, name)(fake, fake, 1, fake, fake, 4, 2, 4, 64, 200, fake, pt, stride, log2, None) != 0
        assert b"page" in lib.rstnet_last_error()
