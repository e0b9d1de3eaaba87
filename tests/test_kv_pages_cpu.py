"""Paged KV cache, the parts that need no GPU: the host page allocator, the C ABI's declarations and argument checks,
the pool sizing and `offline synthesize --kv-gb`."""
import os

import numpy as np
import pytest

from rstnet_b200 import _lib
from rstnet_b200._lib import RstnetError
from rstnet_b200.lm import KV_PAGE, Config, KVPages, kv_page_bytes, kv_pages_for_budget

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("rstnet_lm_rope_kv_append_paged_bf16", "rstnet_lm_paged_decode_attention_bf16")


def test_allocator_lowest_first_replace_release():
    a = KVPages(10, 3, 16, 40)              # 3 pages per ring, the last one half used
    assert a.stride == 3 and a.log2_page == 4 and a.free == 10
    assert a.reserve([0, 1], [20, 5]) == [0, 1]
    assert a.table[0].tolist() == [0, 1, -1] and a.table[1].tolist() == [2, -1, -1] and a.free == 7
    assert a.limit[0] == 20 and a.limit[1] == 5
    a.reserve([2], 1000)                    # beyond the ring: the whole ring, no limit
    assert a.table[2].tolist() == [3, 4, 5] and a.limit[2] == np.iinfo(np.int64).max
    a.release([0])
    assert a.table[0].tolist() == [-1, -1, -1] and a.free == 6 and a.limit[0] == 0
    a.reserve([1], 40)                      # grows in place: page 2 stays, the lowest free pages join
    assert a.table[1].tolist() == [2, 0, 1]
    a.reserve([1], 10)                      # shrinks: keeps its first page
    assert a.table[1].tolist() == [2, -1, -1] and a.free == 6
    a.reserve([0], 48)
    assert a.table[0].tolist() == [0, 1, 6]


def test_failed_reservation_changes_nothing():
    a = KVPages(5, 3, 16, 40)
    a.reserve([0], 33)
    snap = (a.table.copy(), a.held.copy(), a.limit.copy(), a.free)
    for streams, pos in (([1, 2], [40, 40]), ([1], -1), ([0, 0], 1), ([3], 1)):
        with pytest.raises(RstnetError):
            a.reserve(streams, pos)
        assert np.array_equal(a.table, snap[0]) and np.array_equal(a.held, snap[1]) and np.array_equal(a.limit, snap[2])
        assert a.free == snap[3]
    a.reserve([0, 1], [0, 40])              # pages freed by one stream serve another in the same call
    assert a.table[1].tolist() == [0, 1, 2] and a.free == 2


def test_allocator_guard_and_page_sizes():
    a = KVPages(4, 2, 16, 40)
    a.reserve([0], 7)
    a.check([0], [6], 1)
    with pytest.raises(RstnetError):
        a.check([0], [6], 2)
    with pytest.raises(RstnetError):
        a.check([1], [0], 1)                # no pages: no position
    for page in (8, 24, 8192):
        with pytest.raises(RstnetError):
            KVPages(4, 2, page, 40)
    with pytest.raises(RstnetError):
        KVPages(0, 2, 16, 40)


def test_symbols_declared_and_bound():
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    for name in NEW:
        assert f"int {name}(" in header and name in _lib.SYMBOLS
    assert f"#define RSTNET_KV_LOG2_PAGE_MIN {_lib.KV_LOG2_PAGE_MIN}" in header
    assert f"#define RSTNET_KV_LOG2_PAGE_MAX {_lib.KV_LOG2_PAGE_MAX}" in header
    lib = _lib.lib()
    assert lib.rstnet_version() == 206
    for name in NEW:
        assert getattr(lib, name).argtypes


def test_paged_entry_points_check_page_arguments():
    """Every bad page argument returns an error before a launch (so these calls run without a GPU)."""
    lib = _lib.lib()
    fake = 256                              # a pointer the checks never dereference
    for pt, stride, log2 in ((None, 3, 4), (fake, 3, 3), (fake, 3, 13), (fake, 2, 4), (fake, 0, 4)):
        assert lib.rstnet_lm_rope_kv_append_paged_bf16(fake, fake, fake, 64, 64, fake, 1, None, None, fake, fake, 2, 2, 4, 4, 64,
                                                       40, pt, stride, log2, None) != 0
        assert b"page" in lib.rstnet_last_error()
        assert lib.rstnet_lm_paged_decode_attention_bf16(fake, fake, fake, 1, None, None, fake, 2, 2, 4, 4, 64, 40, 40, pt, stride,
                                                         log2, None) != 0
        assert b"page" in lib.rstnet_last_error()


def test_pool_sizing_and_synthesize_kv_gb():
    from rstnet_b200.offline import build_parser
    c = Config(n_layer=32, n_embd=4096, n_head=32, head_size=128, context=2048)
    assert kv_page_bytes(c) == 32 * 2 * 32 * KV_PAGE * 128 * 2 == 32 * 2 ** 20    # 0.5 MiB per position at 7B MHA
    assert kv_pages_for_budget(c, 40) == 1280 and kv_pages_for_budget(c, 0.1) == 3
    base = ["synthesize", "--input", "a", "--config", "b", "--checkpoint", "c", "--output-file", "d"]
    assert build_parser().parse_args(base).kv_gb is None
    assert build_parser().parse_args(base + ["--kv-gb", "40.5"]).kv_gb == 40.5
    for bad in ("0", "-1", "nan", "x"):
        with pytest.raises(SystemExit):
            build_parser().parse_args(base + ["--kv-gb", bad])
