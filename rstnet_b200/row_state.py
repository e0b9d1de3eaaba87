"""One batch row's streaming state as a packed blob in pinned host memory: the segment tables of
`rstnet_segments_gather` / `rstnet_segments_scatter` (csrc/row_state.cu) and the `SessionState` of a suspended duplex
session (serve.DuplexEngine.suspend_rows / resume_rows).

Every layer that keeps per-row state lists it as REGIONS: (name, segments), where segments is an int64 array [k, 4] of
(device address, stride bytes, bytes, count) rows that fill the region back to back, in the layer's canonical order.  A
region's bytes do not depend on the buffer layout it was read from (time- or batch-major codec buffers, contiguous or
paged LM KV), so a blob restores into any row of any engine whose regions have the same names and sizes.  Regions start
at 16-byte offsets of the blob, so the kernel moves them 16 bytes at a time wherever the device side allows it.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from ._lib import RstnetError

SEGMENT_DTYPE = np.dtype({"names": ["base", "stride_bytes", "bytes", "count", "staging_offset"],
                          "formats": ["<u8", "<i8", "<i8", "<i4", "<i8"],
                          "offsets": [0, 8, 16, 24, 32], "itemsize": C.sizeof(_lib.Segment)})
ALIGN = 16


def segs(*rows) -> np.ndarray:
    """(address, stride bytes, bytes, count) rows -> int64 [k, 4]"""
    return np.asarray(rows, dtype=np.int64).reshape(-1, 4)


def tensor_segs(t: torch.Tensor) -> np.ndarray:
    """the whole of a contiguous tensor (a view of one row of a buffer) as one piece"""
    if not t.is_contiguous():
        raise RstnetError("a state segment must be contiguous")
    n = t.numel() * t.element_size()
    return segs((t.data_ptr(), n, n, 1))


def region_bytes(s: np.ndarray) -> int:
    return int((s[:, 2] * s[:, 3]).sum()) if len(s) else 0


def signature(regions) -> Tuple[Tuple[str, int], ...]:
    return tuple((name, region_bytes(s)) for name, s in regions)


def layout(regions) -> Tuple[np.ndarray, int]:
    """-> (the segment table of `regions`, a structured SEGMENT_DTYPE array, and the blob size in bytes)"""
    rows, offs, pos = [], [], 0
    for _, s in regions:
        if len(s):
            sizes = s[:, 2] * s[:, 3]
            offs.append(pos + np.concatenate(([0], np.cumsum(sizes)[:-1])))
            rows.append(s)
            pos += int(sizes.sum())
        pos = -(-pos // ALIGN) * ALIGN
    table = np.zeros(sum(len(r) for r in rows), dtype=SEGMENT_DTYPE)
    if rows:
        allr = np.concatenate(rows)
        table["base"] = allr[:, 0].astype(np.uint64)
        table["stride_bytes"], table["bytes"], table["count"] = allr[:, 1], allr[:, 2], allr[:, 3]
        table["staging_offset"] = np.concatenate(offs)
    return table, pos


def pinned_table(table: np.ndarray) -> torch.Tensor:
    """the table in pinned host memory, which the kernel reads directly (no upload, no synchronise for the checks)"""
    return torch.from_numpy(table.view(np.uint8).copy()).pin_memory()


def run(direction: str, table: torch.Tensor, n: int, blob: torch.Tensor, stream: torch.cuda.Stream, ctas: int) -> None:
    fn = _lib.lib().rstnet_segments_gather if direction == "gather" else _lib.lib().rstnet_segments_scatter
    _lib.check(fn(table.data_ptr(), int(n), blob.data_ptr(), int(ctas), stream.cuda_stream), f"segments_{direction}")


@dataclass
class SessionState:
    """A suspended session: its row's state packed into `blob` (pinned host memory, `nbytes` bytes), the host fields that
    go with it, and the key of the engines it restores into.  Produced by an engine's `suspend_rows`, consumed by
    `resume_rows` of the same engine or of another one with the same key; an incompatible engine raises RstnetError.  The
    blob is valid once `ready` has passed (resume_rows orders itself after it).  It may be larger than `nbytes` (a pooled
    blob).  A resume consumes the state: its blob goes back to the resuming engine's pool, and `blob` becomes None."""
    key: Tuple
    regions: Tuple[Tuple[str, int], ...]
    blob: torch.Tensor
    nbytes: int
    host: Dict[str, Any] = field(default_factory=dict)
    ready: Optional[torch.cuda.Event] = None
    _table: Optional[torch.Tensor] = None     # the gather's segment table, alive until `ready` has passed

    @property
    def positions(self) -> int:
        """the LM positions the session has run (its KV holds min(positions, context) slots)"""
        return int(self.host["pos"])


def check_compatible(state: SessionState, key: Tuple, regions: Sequence) -> None:
    if not isinstance(state, SessionState):
        raise RstnetError(f"expected a SessionState, got {type(state).__name__}")
    if state.key != key:
        diff = [f"{a!r} != {b!r}" for a, b in zip(state.key, key) if a != b] or ["key length"]
        raise RstnetError("this session state belongs to an incompatible engine: " + "; ".join(diff[:3]))
    sig = signature(regions)
    if sig != state.regions:
        bad = next((f"{a} != {b}" for a, b in zip(state.regions, sig) if a != b), "region count")
        raise RstnetError(f"this session state does not fit the engine's rows: {bad}")
