"""CPU oracle of nucleus (top-p) sampling: the kept set of sample_top_p, restated in float64.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): never imported by rstnet_b200/.

Reference: MLLM_v2/utils/sampling.py:66-82 (sample_top_p) on probs = softmax(logits / temp) (sample_token, :85-105).
sample_top_p sorts the probabilities descending, masks every entry whose exclusive cumulative mass exceeds p
(`probs_sum - probs_sort > p`) and renormalises the rest.  Restated here without the fp32 cumsum: the ids < n_valid in
the order (logit desc, index asc), w = exp((l - max) / temp), id kept iff the float64 mass before it is <= p * sum(w).
Ties at the cut are kept lowest index first (torch.sort leaves their order open).  A restricted candidate set (n_valid <
the row length) is the distribution renormalised over the ids < n_valid; the reference's masked samplers
(sample_token_audio[_2048]) give NaN there instead.  Pinned against the unmodified reference by
oracle/gen_golden_sampling.py (tests/golden/sampling_top_p.npz).

The logit rows are a counter-based function of (seed, kind, scale) -- splitmix64 over the index, so the fixture holds no
logits and any numpy reproduces them -- rounded to bf16 as the LM head writes them.
"""
from __future__ import annotations

import numpy as np
import torch

M64 = (1 << 64) - 1


def _splitmix64(x: np.ndarray) -> np.ndarray:
    x = (x + np.uint64(0x9E3779B97F4A7C15)) & np.uint64(M64)
    x = ((x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & np.uint64(M64)
    x = ((x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & np.uint64(M64)
    return x ^ (x >> np.uint64(31))


def uniform(seed: int, n: int) -> np.ndarray:
    """n uniforms in (0, 1), float64, a function of (seed, index) only"""
    with np.errstate(over="ignore"):
        x = _splitmix64(np.arange(n, dtype=np.uint64) + np.uint64(seed) * np.uint64(0x100000001B3))
    return ((x >> np.uint64(11)).astype(np.float64) + 0.5) * (1.0 / (1 << 53))


def logit_row(seed: int, V: int, kind: str, scale: float, temp: float = 1.0, p: float = 0.5) -> torch.Tensor:
    """A bf16 logit row [V].  kind 'gumbel': scale * Gumbel noise (a heavy upper tail, as LM heads have);
    'coarse': the same rounded to multiples of scale / 2 (thousands of exact ties at every cut);
    'tail': 'gumbel' with the upper half of the ids at -inf;
    'planted': 'gumbel' with the 8 ids ranked after the (temp, p) cut raised to the cut id's logit (ties at the cut)."""
    u = uniform(seed, V)
    x = scale * -np.log(-np.log(u))
    if kind == "coarse":
        x = np.round(x * 2.0 / scale) * (scale / 2.0)
    elif kind == "tail":
        x[V // 2:] = -np.inf
    elif kind not in ("gumbel", "planted"):
        raise ValueError(kind)
    row = torch.from_numpy(x).to(torch.bfloat16)
    if kind == "planted":
        order, before, _ = nucleus(row, V, temp)
        r = int((before <= p).sum()) - 1
        row[torch.from_numpy(order[r + 1:r + 9].copy())] = row[int(order[r])].item()
    return row


def nucleus(logits, n_valid: int, temp: float):
    """-> (order [n] ids in (logit desc, index asc), mass_before [n] / Z, w [n] / Z), float64, over the ids < n_valid"""
    x = torch.as_tensor(logits).to(torch.float64).numpy()[:n_valid]
    order = np.lexsort((np.arange(n_valid), -x))
    finite = x[order] > -np.inf
    w = np.where(finite, np.exp((x[order] - x[order[0]]) / temp), 0.0)
    z = w.sum()
    before = np.concatenate([[0.0], np.cumsum(w)[:-1]])
    return order, before / z, w / z


def kept_set(logits, n_valid: int, temp: float, p: float, margin: float = 0.0) -> np.ndarray:
    """bool [n_valid]: the ids sample_top_p keeps (mass before <= p, as fractions of the total); margin > 0 widens the set
    by the ids whose mass before is within margin above p, margin < 0 narrows it."""
    order, before, _ = nucleus(logits, n_valid, temp)
    keep = np.zeros(n_valid, dtype=bool)
    keep[order[before <= p + margin]] = True
    keep[order[0]] = True
    return keep


def kept_probs(logits, n_valid: int, temp: float, p: float) -> np.ndarray:
    """float64 [n_valid]: the renormalised nucleus distribution (0 outside the kept set)"""
    order, before, w = nucleus(logits, n_valid, temp)
    k = before <= p
    k[0] = True
    out = np.zeros(n_valid)
    out[order[k]] = w[k] / w[k].sum()
    return out
