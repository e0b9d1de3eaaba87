"""CPU tests of forced tokens during generation: the aligned-mask to step-layout mapping (`moshi.force_from_aligned`)
against `prompt_from_aligned` and a hand-written loop, the argument checks of the C entry point, `forward_step(force=)`,
`LMGen.step(force=)`, `moshi.generate_many(force=)` and `InferenceImp.generate_many(forced=)`, the new symbol's
declaration, binding and export, and `offline continue --force`."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from rstnet_b200 import _lib
from rstnet_b200._lib import RstnetError
from rstnet_b200.infer import InferenceImp
from rstnet_b200.lm import _LMState
from rstnet_b200.moshi import LMGen, _forced_steps, force_from_aligned, generate_many, prompt_from_aligned

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DELAYS = (0, 0, 1, 1, 0, 1, 1)     # K = 7, dep_q = 3: text and codebook 1 undelayed, as Moshi's [0, 0, 1, ...]
DEP_Q = 3


def _aligned(L, seed):
    return torch.randint(0, 60, (len(DELAYS), L), generator=torch.Generator().manual_seed(seed))


def test_force_mapping_by_hand():
    """delays [0, 0, 1, 1]: a codebook with delay 1 is sampled one step after its aligned frame, so step 0 never takes it"""
    seq = torch.arange(7 * 4).view(7, 4)
    mask = torch.tensor([[1, 0, 1, 0], [0, 1, 0, 0], [1, 1, 1, 1], [0, 0, 0, 1]], dtype=torch.bool)
    want = torch.tensor([[0, -1, 2, -1],
                         [-1, 5, -1, -1],
                         [-1, 8, 9, 10],       # frame 3 would be step 4: past the item's last step
                         [-1, -1, -1, -1]])    # frame 3 of a delayed codebook: no step
    assert torch.equal(force_from_aligned(seq, mask, DELAYS, DEP_Q), want)


@pytest.mark.parametrize("P", [0, 1, 2, 5, 9])
def test_full_mask_agrees_with_prompt_from_aligned(P):
    seq = _aligned(9, P)
    full = force_from_aligned(seq, torch.ones(DEP_Q + 1, 9, dtype=torch.bool), DELAYS, DEP_Q)
    assert full.dtype == torch.int64 and full.shape == (DEP_Q + 1, 9)
    assert torch.equal(full[:, :P], prompt_from_aligned(seq, P, DELAYS, DEP_Q, initial=-1)[:DEP_Q + 1])


def test_partial_mask_vs_hand_loop():
    seq = _aligned(11, 3)
    mask = torch.rand(DEP_Q + 1, 11, generator=torch.Generator().manual_seed(1)) < 0.5
    got = force_from_aligned(seq, mask, DELAYS, DEP_Q)
    for k in range(DEP_Q + 1):
        for t in range(11):
            f = t - DELAYS[k]
            want = int(seq[k, f]) if f >= 0 and bool(mask[k, f]) else -1
            assert int(got[k, t]) == want, (k, t)


def test_force_mapping_rejects_bad_masks():
    seq = _aligned(5, 0)
    ok = torch.ones(DEP_Q + 1, 5, dtype=torch.bool)
    for mask in [ok[:, :4], ok[:3], ok.long(), ok[0], None, np.ones((4, 5), dtype=bool)]:
        with pytest.raises(RstnetError, match="force mask"):
            force_from_aligned(seq, mask, DELAYS, DEP_Q)
    with pytest.raises(RstnetError):
        force_from_aligned(seq.float(), ok, DELAYS, DEP_Q)
    with pytest.raises(RstnetError):
        force_from_aligned(seq, ok, DELAYS[:6], DEP_Q)


def test_generate_many_forced_item_checks():
    seq = _aligned(6, 2)
    vocab = (60, 50, 50, 50)
    ok = torch.zeros(DEP_Q + 1, 6, dtype=torch.bool)
    ok[1] = True
    assert _forced_steps("u", seq.clamp(max=49), ok, DELAYS, DEP_Q, vocab).shape == (DEP_Q + 1, 6)
    with pytest.raises(RstnetError, match="'u'.*force mask"):
        _forced_steps("u", seq, ok[:, :5], DELAYS, DEP_Q, vocab)          # a mask of the wrong length
    big = seq.clamp(max=49)
    big[1, 2] = 50
    with pytest.raises(RstnetError, match="'u'.*outside"):
        _forced_steps("u", big, ok, DELAYS, DEP_Q, vocab)
    big[1, 2] = -1
    with pytest.raises(RstnetError, match="outside"):
        _forced_steps("u", big, ok, DELAYS, DEP_Q, vocab)
    ok2 = ok.clone()
    ok2[1, 2] = False
    _forced_steps("u", big, ok2, DELAYS, DEP_Q, vocab)                # an id that is not forced is not checked


def _small_lm():
    from rstnet_b200.moshi import LMModel
    return LMModel(delays=list(DELAYS), n_q=6, dep_q=DEP_Q, card=60, text_card=500, dim=64, num_heads=2, num_layers=1,
                   hidden_scale=4.125, norm="rms_norm_f32", gating="silu", positional_embedding="rope", depformer_dim=64,
                   depformer_dim_feedforward=128, depformer_num_heads=2, depformer_num_layers=1, depformer_multi_linear=True,
                   depformer_weights_per_step=True, depformer_pos_emb="none", existing_text_padding_id=3, context=16)


def test_moshi_force_argument_errors():
    gen = LMGen(_small_lm(), use_sampling=False)
    with pytest.raises(RstnetError, match="force must be a dict"):
        next(generate_many(gen, [], 2, force=[1]))
    # LMGen.step(force=) takes input_tokens' convention [B, dep_q + 1, 1]; a stand-in scope of 2 rows checks it first
    calls = []
    gen._st = SimpleNamespace(B=2, lm=SimpleNamespace(set_force=calls.append))
    x = torch.zeros(2, 3, 1, dtype=torch.int64)
    for bad in [torch.zeros(2, 4, dtype=torch.int64), torch.zeros(2, 4, 2, dtype=torch.int64), [[-1] * 4] * 2]:
        with pytest.raises(RstnetError, match="force"):
            gen.step(x, force=bad)
    assert calls == []


def test_set_force_argument_errors():
    st = SimpleNamespace(B=3, c=SimpleNamespace(dep_q=8), force_rows=torch.full((3, 9), -1, dtype=torch.int32))
    for bad in [torch.zeros(3, 8, dtype=torch.int64), torch.zeros(2, 9, dtype=torch.int64), torch.zeros(3, 9),
                torch.zeros(3, 9, dtype=torch.bool), np.zeros((3, 9), dtype=np.int64)]:
        with pytest.raises(RstnetError, match="force is an integer tensor"):
            _LMState.set_force(st, bad)
    _LMState.set_force(st, torch.tensor([[5] + [-1] * 8] * 3))
    assert st.force_rows[:, 0].tolist() == [5, 5, 5] and bool((st.force_rows[:, 1:] == -1).all())


class _FakeGPT:
    """what the argument checks of InferenceImp.generate_many read of the model (no scope is ever opened)"""
    config = SimpleNamespace(padded_vocab_size=1000, audio_card=2050, context=64)
    num_codebooks = 9

    def reserve_kv(self, *a):
        raise AssertionError("a scope was opened")


def _tts(P, G):
    seq = torch.zeros(9, P + G, dtype=torch.int64)
    seq[0, P:] = 128002
    return seq


def test_generate_many_forced_checks_raise_before_any_launch():
    imp = InferenceImp(None, _FakeGPT(), "sampling", 0.7, 25, 0.8, 30, "TTS")
    items = [("a", _tts(4, 5)), ("b", _tts(3, 2))]
    ok = torch.full((9, 5), -1, dtype=torch.int64)
    assert imp._check_forced("a", ok, 5).dtype == np.int32
    bad = {"shape": ok[:, :4], "rows": ok[:8], "dtype": ok.int(), "float": ok.float(), "list": ok.tolist()}
    for name, f in bad.items():
        with pytest.raises(RstnetError, match="'a'.*int64"):
            imp._check_forced("a", f, 5)
    for row, v in [(0, 1000), (1, 2050), (5, -2)]:
        f = ok.clone()
        f[row, 2] = v
        with pytest.raises(RstnetError, match="'a'.*vocabulary"):
            imp._check_forced("a", f, 5)
    f = ok.clone()
    f[0, 0], f[1, 1], f[8, 4] = 999, 2049, 0
    imp._check_forced("a", f, 5)                                  # ids outside the candidate sets are allowed
    with pytest.raises(RstnetError, match="not among the items"):
        next(imp.generate_many(items, 2, forced={"a": ok, "zz": ok}))
    with pytest.raises(RstnetError, match="dict"):
        next(imp.generate_many(items, 2, forced=[ok]))
    # an item's table is checked when the item is read: for a lazily read corpus the first bad table raises there
    pull = imp._puller(iter(items), None, None, forced={"a": ok[:, :3]}, tables={})
    with pytest.raises(RstnetError, match="'a'"):
        pull()
    tables = {}
    pull = imp._puller(iter(items), None, None, forced={"b": torch.full((9, 2), 7)}, tables=tables)
    pull(), pull()
    assert list(tables) == ["b"] and tables["b"].dtype == np.int32
    pull = imp._puller(iter(items), None, None, forced={"q": ok}, tables={})
    pull(), pull()
    with pytest.raises(RstnetError, match="not among the items"):
        pull()


def test_abi_declares_binds_and_exports_force_tokens():
    header = open(os.path.join(ROOT, "include", "rstnet_b200.h")).read()
    name = "rstnet_lm_force_tokens"
    assert f"int {name}(" in header and name in _lib.SYMBOLS
    lib = _lib.lib()
    assert len(getattr(lib, name).argtypes) == 8 and lib.rstnet_version() == 206
    integration = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    assert name in integration and "added in version 206, no version change" in integration.lower()


@pytest.mark.parametrize("bad,msg", [
    (dict(tokens=None), b"null pointer"), (dict(force=None), b"null pointer"), (dict(rows=0), b"bad shape"),
    (dict(V=0), b"bad shape"), (dict(col=-1), b"bad shape"), (dict(col=9), b"bad shape"), (dict(force_stride=4), b"bad shape"),
])
def test_force_tokens_refuses_bad_arguments(bad, msg):
    """fake (never dereferenced) device pointers: every case is refused before any launch"""
    a = dict(tokens=8, tok_stride=9, col=4, force=8, force_stride=9, rows=3, V=2050)
    a.update(bad)
    before = _lib.launch_count()
    lib = _lib.lib()
    assert lib.rstnet_lm_force_tokens(a["tokens"], a["tok_stride"], a["col"], a["force"], a["force_stride"], a["rows"], a["V"],
                                      None) != 0
    assert msg in lib.rstnet_last_error() and _lib.launch_count() == before


def test_continue_cli_parses_force():
    from rstnet_b200.offline import build_parser
    base = ["continue", "--model", "moshi", "--config", "c.json", "--checkpoint", "ck", "--input", "in.pt", "--output-file",
            "o.pt", "--prompt-frames", "4"]
    assert build_parser().parse_args(base).force is None
    for v in ("text", "audio"):
        assert build_parser().parse_args(base + ["--force", v]).force == v
    with pytest.raises(SystemExit):
        build_parser().parse_args(base + ["--force", "user"])
