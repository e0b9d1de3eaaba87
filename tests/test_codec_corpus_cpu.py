"""Host-side pieces of the codec's corpus batching (no GPU): the new entry point is declared, exported and bound, and the
offline CLI takes --capacity for tokenize and reconstruct without changing what they run when it is absent."""
import os

from rstnet_b200 import _lib, offline

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_rows_fill_tail_is_declared_and_listed():
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    assert "int rstnet_rows_fill_tail_f32(" in header
    assert "rstnet_rows_fill_tail_f32" in _lib.SYMBOLS


def test_cli_capacity_option():
    p = offline.build_parser()
    base = {"tokenize": ["--weights", "w", "--wav-scp", "s", "--output-file", "o"],
            "reconstruct": ["--weights", "w", "--input", "i", "--output", "o"]}
    for cmd, args in base.items():
        assert p.parse_args([cmd, *args]).capacity is None            # the per-clip drivers, as before
        assert p.parse_args([cmd, *args, "--capacity", "96"]).capacity == 96
