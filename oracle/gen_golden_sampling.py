"""Generate tests/golden/sampling_top_p.npz by running the UNMODIFIED reference's nucleus sampler here.

Run:  python -m oracle.gen_golden_sampling      (needs a checkout of the reference repository at REF)

For seeded bf16 logit rows (oracle/sampling_oracle.logit_row: V = 2 050 with 2 048 / 2 049 / 2 050 candidates, 32 000
and 152 064; several temperatures; p in {0.1, 0.5, 0.9, 0.99}; rows with thousands of ties, with -inf tails and with
ties planted at the cut) it calls the reference's `sample_top_p(softmax(logits[:n_valid] / temp), p)` and records the
sorted, masked, renormalised `probs_sort` that sample_top_p hands to `multinomial`, by wrapping the module-level
`multinomial` it calls (the reference's code is not changed).  The fixture keeps, per row: the kept ids (nonzero entries
of probs_sort, mapped back through the same descending torch.sort of the same probs) as a bit mask, their count and the
16 largest renormalised probabilities.  The logits themselves are a function of the stored row parameters.
"""
from __future__ import annotations

import hashlib
import os
import sys

sys.dont_write_bytecode = True

import numpy as np
import torch

from . import sampling_oracle as O
from .gen_golden_lm import GOLDEN, REF

PS = (0.1, 0.5, 0.9, 0.99)


def rows():
    """(seed, V, n_valid, kind, scale, temp, p) of every fixture row"""
    out = []
    seed = 100
    for V, n_valids in ((2050, (2048, 2049, 2050)), (32000, (32000,)), (152064, (152064,))):
        for i, p in enumerate(PS):
            for kind, scale in (("gumbel", 1.5), ("coarse", 1.0), ("planted", 0.8)):
                temp = (0.7, 1.0, 1.3)[(i + len(out)) % 3]
                out.append((seed, V, n_valids[(i + len(out)) % len(n_valids)], kind, scale, temp, p))
                seed += 1
        out.append((seed, V, n_valids[0], "tail", 1.0, 0.8, 0.9))
        seed += 1
    return out


def row_logits(seed, V, n_valid, kind, scale, temp, p) -> torch.Tensor:
    return O.logit_row(seed, V, kind, scale, temp=temp, p=p)


def main():
    sys.path.insert(0, REF)
    import utils.sampling as S

    seen = {}
    orig = S.multinomial

    def recording_multinomial(input, num_samples, replacement=False, *, generator=None):
        seen["probs_sort"] = input.detach().clone()
        return orig(input, num_samples, replacement, generator=generator)

    S.multinomial = recording_multinomial
    spec = rows()
    masks, counts, tops, digests = [], [], [], []
    Vmax = max(r[1] for r in spec)
    try:
        for r in spec:
            seed, V, n_valid, kind, scale, temp, p = r
            lg = row_logits(*r)
            probs = torch.softmax(lg[:n_valid].float() / temp, dim=-1)
            _, idx = torch.sort(probs, dim=-1, descending=True)   # the sort sample_top_p runs on the same probs
            seen.clear()
            S.sample_top_p(probs.clone(), p)
            ps = seen["probs_sort"]
            kept = idx[ps > 0].numpy()
            m = np.zeros(Vmax, dtype=bool)
            m[kept] = True
            masks.append(np.packbits(m))
            counts.append(len(kept))
            tops.append(ps[:16].double().numpy())
            digests.append(hashlib.sha256(lg.view(torch.int16).numpy().tobytes()).hexdigest()[:16])
    finally:
        S.multinomial = orig
    path = os.path.join(GOLDEN, "sampling_top_p.npz")
    np.savez_compressed(path,
                        seed=np.array([r[0] for r in spec], dtype=np.int64), V=np.array([r[1] for r in spec], dtype=np.int64),
                        n_valid=np.array([r[2] for r in spec], dtype=np.int64), kind=np.array([r[3] for r in spec]),
                        scale=np.array([r[4] for r in spec]), temp=np.array([r[5] for r in spec]),
                        p=np.array([r[6] for r in spec]), kept_bits=np.stack(masks), n_kept=np.array(counts, dtype=np.int64),
                        top_probs=np.stack(tops), logits_sha=np.array(digests))
    print(path, os.path.getsize(path), "bytes,", len(spec), "rows; kept counts", counts)


if __name__ == "__main__":
    main()
