"""Best-of-N TTS, the parts that need no GPU: KVPages sharing (reference counts, copy-on-write, all or nothing), the
page allocator without sharing against a restatement of the reservation-only allocator, sample_seed, the argument
checks of generate_many(n_samples=...), stream_many and TTSEngine, the new C entry point's declaration and argument
checks, and the offline CLI flags."""
import heapq
import os

import numpy as np
import pytest
import torch

from rstnet_b200 import _lib
from rstnet_b200._lib import RstnetError
from rstnet_b200.infer import Candidate, InferenceImp, rank_candidates, sample_seed
from rstnet_b200.lm import KVPages
from rstnet_b200.serve import TTSEngine

from test_tts_batch_cpu import FakeGPT, _utt
from test_tts_stream_cpu import FakeCodec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("rstnet_kv_pages_copy",)


class ReservationOnly:
    """The page allocator as it is without sharing: one owner per page, lowest free page first."""

    def __init__(self, n_pages, streams, page, cap):
        self.page, self.cap = page, cap
        self.stride = -(-cap // page)
        self.table = np.full((streams, self.stride), -1, dtype=np.int32)
        self.held = np.zeros(streams, dtype=np.int64)
        self.free = list(range(n_pages))

    def reserve(self, streams, positions):
        need = [-(-min(p, self.cap) // self.page) for p in positions]
        grow = sum(max(0, n - int(self.held[x])) for x, n in zip(streams, need))
        shrink = sum(max(0, int(self.held[x]) - n) for x, n in zip(streams, need))
        if grow > len(self.free) + shrink:
            raise RstnetError("short")
        for x, n in zip(streams, need):
            for page in self.table[x, n:self.held[x]]:
                heapq.heappush(self.free, int(page))
            self.table[x, n:] = -1
        for x, n in zip(streams, need):
            for i in range(int(self.held[x]), n):
                self.table[x, i] = heapq.heappop(self.free)
            self.held[x] = n

    def detach(self, s):
        pages = [int(p) for p in self.table[s, :self.held[s]]]
        self.table[s] = -1
        self.held[s] = 0
        return pages

    def give_back(self, pages):
        for p in pages:
            heapq.heappush(self.free, int(p))


def test_without_share_tables_and_free_lists_are_unchanged():
    """a recorded sequence of admissions, growths, releases and suspends gives the same tables and free heap, step by step"""
    rng = np.random.default_rng(3)
    a, b = KVPages(40, 6, 16, 100), ReservationOnly(40, 6, 16, 100)
    parked = []
    for step in range(400):
        op = rng.integers(0, 4)
        s = [int(x) for x in rng.choice(6, size=int(rng.integers(1, 4)), replace=False)]
        pos = [int(x) for x in rng.integers(0, 140, size=len(s))]
        if op <= 1:
            try:
                b.reserve(s, pos)
            except RstnetError:
                with pytest.raises(RstnetError):
                    a.reserve(s, pos)
            else:
                a.reserve(s, pos)
        elif op == 2:
            a.release(s)
            b.reserve(s, [0] * len(s))
        elif parked and rng.integers(0, 2):
            a.give_back(parked[-1][0])
            b.give_back(parked.pop()[1])
        else:
            parked.append((a.detach(s[0]), b.detach(s[0])))
        assert np.array_equal(a.table, b.table) and a._free == b.free, step
        assert not a.sharing and not a.spares and int(a.refs.max()) <= 1
        assert a.cow(range(6), np.zeros(6, dtype=np.int64), 1) == ([], [])


def test_share_maps_full_pages_copies_the_partial_one_and_counts_references():
    a = KVPages(20, 4, 16, 128)            # 8 pages per ring, no wrap below 128 positions
    a.reserve([0], 40)                     # pages 0, 1, 2: the prompt writes 37 positions (2 full pages + 5 slots)
    free0 = a.free
    pairs, rows = a.share(0, [1, 2], 40, written=37)
    assert rows == [1, 2]
    # full pages 0 and 1 shared; page 2 (slots 32..47) is written first at 37: each dst gets its own copy
    assert a.table[1, :3].tolist() == [0, 1, 3] and a.table[2, :3].tolist() == [0, 1, 4]
    assert pairs == [(2, 3), (2, 4)]
    assert a.refs[0] == a.refs[1] == 3 and a.refs[2] == a.refs[3] == a.refs[4] == 1
    assert a.free == free0 - 2 and a.in_use == 5 and a.held[1] == 3 and a.limit[1] == 40
    # a page returns to the heap exactly when its last reference goes
    a.release([0])
    assert a.refs[0] == 2 and 0 not in a._free and 2 in a._free
    a.release([1])
    assert a.refs[0] == 1 and 0 not in a._free and 3 in a._free
    a.release([2])
    assert a.refs[0] == 0 and {0, 1, 4} <= set(a._free) and a.free == 20
    # detach keeps the references until give_back
    a.reserve([0], 32)
    a.share(0, [3], 64, written=32)        # at a page boundary: nothing to copy, page 2 is the dst's own
    assert a.table[3, :4].tolist() == [0, 1, 2, 3]
    pages = a.detach(3)
    a.release([0])
    assert a.refs[0] == 1 and 0 not in a._free
    a.give_back(pages)
    assert a.free == 20 and int(a.refs.max()) == 0


def test_share_is_all_or_nothing():
    a = KVPages(6, 4, 16, 128)
    a.reserve([0], 40)                     # 3 pages; 3 free
    a.reserve([3], 16)                     # 1 page; 2 free
    snap = (a.table.copy(), a.held.copy(), a.limit.copy(), list(a._free), a.refs.copy())
    for args in ((0, [1, 2], 64, 37),      # 2 x (1 copy + 1 new page) = 4 > 2
                 (0, [1], 200, 37),        # beyond the ring: the whole ring
                 (0, [3], 40, 37),         # the dst holds pages
                 (0, [1], 30, 37),         # positions < written
                 (0, [0], 40, 37), (0, [5], 40, 37)):
        with pytest.raises(RstnetError):
            a.share(*args[:3], written=args[3])
        assert all(np.array_equal(x, y) for x, y in zip(snap[:3], (a.table, a.held, a.limit)))
        assert a._free == snap[3] and np.array_equal(a.refs, snap[4]) and not a.spares


def test_copy_on_write_exactly_when_the_written_page_is_shared():
    cap, page = 64, 16                     # 4 pages per ring
    a = KVPages(40, 4, page, cap)
    a.reserve([0], 100)                    # src: the whole ring (it wraps too)
    pairs, _ = a.share(0, [1, 2], 100, written=40)   # full pages 0, 1 shared; page 2 copied now; page 3 own
    assert pairs == [(2, 4), (2, 6)] and a.table[1].tolist() == [0, 1, 4, 5] and a.table[2].tolist() == [0, 1, 6, 7]
    # every stream writes positions 40 .. 99: slots 40..63, then 0..35 -- pages 0 and 1 again.  3 holders, 3 writers:
    # 2 copies of each set aside (the last writer keeps the original)
    assert {k: len(v) for k, v in a.spares.items()} == {0: 2, 1: 2}
    free_before = a.free
    for p in range(40, 64):                # no shared page in slots 40..63
        assert a.cow([0, 1, 2], [p] * 3, 1) == ([], [])
    pairs, rows = a.cow([1], [64], 1)      # position 64 -> slot 0: page 0 is shared -> stream 1 copies it
    assert len(pairs) == 1 and pairs[0][0] == 0 and rows == [1] and a.table[1, 0] == pairs[0][1]
    assert a.refs[0] == 2 and len(a.spares[0]) == 1 and a.free == free_before
    assert a.cow([1], [65], 1) == ([], [])  # its own copy now
    pairs, rows = a.cow([0, 2], [64, 64], 1)   # src copies, and the last holder (stream 2) keeps the original
    assert len(pairs) == 1 and rows == [0] and a.table[2, 0] == 0 and a.refs[0] == 1 and 0 not in a.spares
    # a stream that leaves returns the spare no one can need any more
    a.release([2])
    assert a.refs[1] == 2 and len(a.spares[1]) == 1
    assert a.sharing                      # page 1 still has two holders
    a.release([0, 1])
    assert a.free == 40 and not a.spares and int(a.refs.max()) == 0 and not a.sharing


def test_sharing_ends_with_the_last_shared_page():
    """once every shared page is down to one holder, writes no longer look for pages to copy"""
    a = KVPages(10, 2, 16, 64)
    a.reserve([0], 20)
    a.share(0, [1], 20, written=16)        # page 0 shared by streams 0 and 1
    assert a.sharing
    a.cow([1], [0], 1)                     # stream 1 writes slot 0: its own copy, page 0 back to one holder
    assert not a.sharing and int(a.refs.max()) == 1


@pytest.mark.parametrize("P,G", [(200, 1900), (300, 1800), (130, 1960), (1000, 1100)])
def test_admission_count_is_what_the_fork_takes_at_7b_shapes(P, G):
    """7B shapes (context 2048, pages of 64), N = 4, prompts of 3 or more pages and P + G >= context: a pool of exactly the
    pages batch TTS counts for the utterance admits it, the fork takes all of them, and every copy at the ring wrap comes
    from the spares set aside, so no write of the generation finds the pool short."""
    from types import SimpleNamespace
    from rstnet_b200.infer import _TTSRows
    N, cap = 4, 2048
    need = _TTSRows.pages_needed(SimpleNamespace(pages=KVPages(10 ** 6, N, 64, cap), n_samples=N), P, G)
    a = KVPages(need, N, 64, cap)
    a.reserve([0], P + G)
    a.share(0, [1, 2, 3], P + G, written=P)
    assert a.free == 0
    copies = 0
    for p in range(P, P + G):
        copies += len(a.cow(range(N), [p] * N, 1)[0])
    wrapped = len(a.written_pages(cap, P + G))     # shared pages reached again at the wrap, each copied by N - 1 holders
    assert copies == (N - 1) * min(wrapped, a.pages_for(P) - (P % 64 != 0)) and a.free == 0
    a.release(range(N))
    assert a.free == need and not a.sharing and not a.spares


def test_copy_on_write_a_held_write_and_a_multi_position_chunk():
    a = KVPages(40, 3, 16, 64)
    a.reserve([0], 20)
    a.share(0, [1], 20, written=16)        # page 0 shared, no copy (at a boundary), page 1 the dst's own
    assert a.cow([0], [0], 1)[0] and a.table[0, 0] != a.table[1, 0]   # a write into slot 0 of a shared page copies it
    b = KVPages(40, 3, 16, 64)
    b.reserve([0], 64)
    b.share(0, [1], 64, written=48)
    pairs, rows = b.cow([1], [60], 8)      # slots 60..63, then 0..3: page 0 shared
    assert [p[0] for p in pairs] == [int(b.table[0, 0])] and rows == [1]


def test_sample_seed():
    for s in (0, 1, 7, 2 ** 31, 2 ** 32 - 1):
        assert sample_seed(s, 0) == s
        keys = [sample_seed(s, i) for i in range(256)]
        assert len(set(keys)) == 256 and all(0 <= k < 2 ** 32 for k in keys)
    assert sample_seed(5, 1) == (5 + 0x9E3779B9) % 2 ** 32
    with pytest.raises(RstnetError):
        sample_seed(0, -1)


def test_rank_candidates():
    z = torch.zeros(8, 1)
    c = [Candidate(0, z, -10.0, -1.0, 5), Candidate(1, z, -5.0, -9.0, 5), Candidate(2, z, -4.0, 0.0, 2),
         Candidate(3, z, -5.0, -2.0, 5)]
    assert [x.index for x in rank_candidates(c, "logprob")] == [1, 3, 0, 2]   # per frame: -1, -1, -2, -2
    assert [x.index for x in rank_candidates(c[::-1], None)] == [0, 1, 2, 3]


def _imp(model):
    return InferenceImp(None, model, "sampling", 0.7, 25, 0.8, 30, "TTS")


def _items():
    return [("u0", _utt(3, 2, 1)), ("u1", _utt(2, 4, 2))]


def test_generate_many_n_samples_argument_checks():
    imp = _imp(FakeGPT())
    for n in (0, -1, 2.0, True, "2"):
        with pytest.raises(RstnetError, match="n_samples must be an int"):
            next(imp.generate_many(_items(), 4, n_samples=n))
    with pytest.raises(RstnetError, match="more than capacity"):
        next(imp.generate_many(_items(), 2, n_samples=3))
    with pytest.raises(RstnetError, match="no paged KV scope"):   # the stand-in has no reserve_kv / fork_kv
        next(imp.generate_many(_items(), 4, n_samples=2))
    with pytest.raises(RstnetError, match="rank"):
        next(imp.generate_many(_items(), 4, rank="mean"))
    # n_samples = 1 is the plain call
    assert [u for u, _ in imp.generate_many(_items(), 2, n_samples=1)] == [u for u, _ in _imp(FakeGPT()).generate_many(_items(), 2)]


def test_streamed_paths_reject_n_samples():
    imp = _imp(FakeGPT())
    with pytest.raises(RstnetError, match="streamed TTS takes n_samples = 1"):
        next(imp.stream_many(_items(), 4, FakeCodec(), n_samples=2))
    with pytest.raises(RstnetError, match="streamed TTS takes n_samples = 1"):
        TTSEngine(imp, FakeCodec(), 4, n_samples=2)
    with pytest.raises(RstnetError, match="n_samples must be an int"):
        TTSEngine(imp, FakeCodec(), 4, n_samples=0)


def test_new_symbols_declared_bound_and_exported():
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert f" {name}(" in header and name in _lib.SYMBOLS, name
    assert "#define RSTNET_KV_COPY_MAX_POOLS 256" in header and _lib.KV_COPY_MAX_POOLS == 256
    from rstnet_b200 import build
    build.build()
    lib = _lib.lib()
    for name in NEW_SYMBOLS:
        assert hasattr(lib, name), name
    assert lib.rstnet_version() == 206


def test_kv_pages_copy_argument_checks_return_before_any_launch():
    """Each call is rejected by a check that needs no device: nothing is dereferenced and no launch is made."""
    import ctypes as C
    lib = _lib.lib()
    fake = 1 << 20
    pools = (C.c_void_p * 2)(fake, fake)
    null_pool = (C.c_void_p * 2)(fake, None)
    pairs = (C.c_int32 * 2)(0, 1)
    n0 = lib.rstnet_launch_count()
    for args, msg in (((None, 2, pairs, 1, 64, 4), "null pools"), ((pools, 2, None, 1, 64, 4), "null pools"),
                      ((pools, 0, pairs, 1, 64, 4), "n_pools"), ((pools, 257, pairs, 1, 64, 4), "n_pools"),
                      ((pools, 2, pairs, -1, 64, 4), "n_pairs"), ((pools, 2, pairs, 1, 0, 4), "page_bytes"),
                      ((pools, 2, pairs, 1, -8, 4), "page_bytes"), ((pools, 2, pairs, 1, 64, 0), "ctas"),
                      ((null_pool, 2, pairs, 1, 64, 4), "pool 1 is a null pointer")):
        assert lib.rstnet_kv_pages_copy(*args, None) != 0, msg
        assert msg in lib.rstnet_last_error().decode(), (msg, lib.rstnet_last_error())
    assert lib.rstnet_kv_pages_copy(pools, 2, pairs, 0, 64, 4, None) == 0   # no pairs: nothing to do
    assert lib.rstnet_launch_count() == n0


def test_synthesize_parser_n_samples():
    from rstnet_b200 import offline
    p = offline.build_parser()
    base = ["synthesize", "--input", "i", "--config", "c", "--checkpoint", "k", "--output-file", "o"]
    a = p.parse_args(base)
    assert a.n_samples == 1 and not a.all_samples
    a = p.parse_args(base + ["--n-samples", "4", "--all-samples"])
    assert a.n_samples == 4 and a.all_samples
