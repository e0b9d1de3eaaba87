"""CPU checks of nucleus sampling and per-row sampling settings: the float64 restatement (oracle/sampling_oracle.py)
against the reference's kept sets (tests/golden/sampling_top_p.npz, oracle/gen_golden_sampling.py), `Sampling`'s
validation, the C entry point's declaration and binding, and the `synthesize` flags."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import sampling_oracle as O
from oracle.gen_golden_sampling import row_logits
from rstnet_b200 import _lib
from rstnet_b200.lm import Sampling

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# The reference cuts on an fp32 cumsum of fp32 probabilities (up to 152 064 terms); the restatement on float64.  Their
# kept counts may differ only at ranks whose float64 mass before is within MARGIN of p (the largest seen: 1.0e-5).
MARGIN = 3e-5


def _rows(golden_dir):
    g = np.load(os.path.join(golden_dir, "sampling_top_p.npz"))
    for j in range(len(g["seed"])):
        r = (int(g["seed"][j]), int(g["V"][j]), int(g["n_valid"][j]), str(g["kind"][j]), float(g["scale"][j]),
             float(g["temp"][j]), float(g["p"][j]))
        yield r, g, j


def test_restatement_gives_the_reference_kept_sets(golden_dir):
    n = 0
    for r, g, j in _rows(golden_dir):
        seed, V, n_valid, kind, scale, temp, p = r
        lg = row_logits(*r)
        assert hashlib.sha256(lg.view(torch.int16).numpy().tobytes()).hexdigest()[:16] == str(g["logits_sha"][j])
        ref = np.unpackbits(g["kept_bits"][j])[:n_valid].astype(bool)
        assert int(ref.sum()) == int(g["n_kept"][j])
        order, before, _ = O.nucleus(lg, n_valid, temp)
        mine = O.kept_set(lg, n_valid, temp, p)
        vals = lg.float().numpy()[:n_valid]
        # both are prefixes of the (logit desc) order: the reference's ties at the cut may be other ids of the same value
        n_ref, n_mine = int(ref.sum()), int(mine.sum())
        assert np.array_equal(np.sort(vals[ref])[::-1], vals[order[:n_ref]]), r
        assert np.array_equal(mine[order[:n_mine]], np.ones(n_mine, dtype=bool)), r
        lo, hi = sorted((n_ref, n_mine))
        assert np.all(np.abs(before[lo:hi] - p) <= MARGIN), (r, n_ref, n_mine)
        # the 16 largest renormalised probabilities sample_top_p handed to multinomial
        probs = np.sort(O.kept_probs(lg, n_valid, temp, p))[::-1][:16]
        np.testing.assert_allclose(probs, g["top_probs"][j], rtol=0, atol=2e-5)
        n += 1
    assert n == 39


def test_fixture_has_ties_at_the_cut(golden_dir):
    """the planted and coarse rows put several ids of the cut's logit on both sides of it"""
    split = 0
    for r, g, j in _rows(golden_dir):
        seed, V, n_valid, kind, scale, temp, p = r
        lg = row_logits(*r)
        keep = O.kept_set(lg, n_valid, temp, p)
        vals = lg.float().numpy()[:n_valid]
        cut = vals[keep].min()
        split += bool((vals[~keep] == cut).any())
    assert split >= 8


@pytest.mark.parametrize("bad", [dict(temp=float("nan")), dict(temp_text=float("inf")), dict(top_p=-0.1), dict(top_p_text=float("nan")),
                                 dict(top_k=1025), dict(top_k_text=2.5), dict(top_k=True), dict(temp="0.7")])
def test_sampling_rejects_bad_values(bad):
    with pytest.raises(_lib.RstnetError):
        Sampling(**bad)


def test_sampling_heads():
    assert Sampling().heads() == ((25, 0.7, 0.0), (30, 0.8, 0.0))
    assert Sampling(use_sampling=False, top_p=0.5).heads() == ((0, 1.0, 0.0), (0, 1.0, 0.0))
    assert Sampling(temp=0.0).heads()[1] == (0, 1.0, 0.0)
    assert Sampling(top_k=0).heads()[1] == (-1, 0.8, 0.0)
    assert Sampling(top_k=-1, top_k_text=-5).heads() == ((-1, 0.7, 0.0), (-1, 0.8, 0.0))   # no top-k, as forward_step reads it
    assert Sampling(top_p=0.9).heads()[1][0] == -1 and abs(Sampling(top_p=0.9).heads()[1][2] - 0.9) < 1e-7
    assert Sampling(top_p_text=1.5).heads()[0] == (-1, 0.7, 0.0)     # keeps every candidate: the multinomial


def test_params_entry_point_declared_and_bound():
    """rstnet_lm_sample_params_bf16 is the sampler's only entry point"""
    src = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    assert "int rstnet_lm_sample_params_bf16(" in src
    assert "rstnet_lm_sample_params_bf16" in _lib.SYMBOLS
    lib = _lib.lib()
    for name in ("rstnet_lm_sample_bf16", "rstnet_lm_sample_rows_bf16"):
        assert name not in src and name not in _lib.SYMBOLS and not hasattr(lib, name), name
    assert lib.rstnet_version() == 206


def test_synthesize_top_p_flags_parse():
    from rstnet_b200.offline import build_parser
    a = build_parser().parse_args(["synthesize", "--input", "i", "--config", "c", "--checkpoint", "k", "--output-file", "o",
                                   "--top-p", "0.9", "--top-p-text", "0.8"])
    assert (a.top_p, a.top_p_text) == (0.9, 0.8)
    a = build_parser().parse_args(["synthesize", "--input", "i", "--config", "c", "--checkpoint", "k", "--output-file", "o"])
    assert (a.top_p, a.top_p_text) == (0.0, 0.0)
