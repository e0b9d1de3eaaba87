"""Generate tests/golden/lm_tasks.npz: the reference generation loop on all four tasks, with its early stop firing.

Run:  python -m oracle.gen_golden_tasks      (needs a checkout of the reference repository at gen_golden_lm.REF)

The UNMODIFIED reference `InferenceImp` (compiled from infer_no_streaming.py as oracle/gen_golden_lm.py does) runs each
item on a reference GPT of the small LM spec (oracle/lm_oracle.SMALL with context = block_size = 64, so that an ASR item,
whose window runs 13 frames past its text, fits the temporal context), in fp32 and bf16, greedy and top-1.  Only its TTS
branch returns: the other branches raise UnboundLocalError at the `gt_audio` test after the loop (:299), which only the
TTS branch binds.  The loop has finished by then, so the generated frames are read from the raising frame's locals --
the audio rows from `final_results`, the text row from `prefix` -- and the raise is asserted to come from that line.

Random weights almost never pick id 2048, so the stop would not fire: row 2048 of the audio heads audio_linears.3..7 is
multiplied by STOP_GAIN (recorded in the fixture).  Every item is also run through oracle/task_oracle.inference_imp,
which must reproduce the reference bit for bit; the windowed TTS items (lengths=, which the reference cannot express)
come from the oracle alone.
"""
from __future__ import annotations

import dataclasses
import os
import sys
import traceback

import numpy as np
import torch

from . import lm_oracle as L
from . import task_oracle as T
from .gen_golden import weights_digest
from .gen_golden_lm import GOLDEN, load_reference_inference_imp, reference_gpt

CFG = dataclasses.replace(L.SMALL, context=L.SMALL.block_size)
WEIGHT_SEED, STOP_GAIN, STOP_HEADS = 7, 1.5, (3, 4, 5, 6, 7)
MODES = (("greedy", False, 0), ("top1", True, 1))


def task_weights(dtype=torch.float32) -> L.W:
    """the fixture's weights: L.synthetic_weights(CFG, seed 7, std 0.05) with row 2048 of audio_linears.3..7 scaled"""
    w = L.synthetic_weights(CFG, seed=WEIGHT_SEED, dtype=torch.float32, std=0.05)
    for k in STOP_HEADS:
        w[f"audio_linears.{k}.weight"][2048] *= STOP_GAIN
    return {k: v.to(dtype) for k, v in w.items()}


def task_sequence(task: str, a: int, b: int, pad: int, seed: int) -> torch.Tensor:
    """A [9, a + b + pad] item of `task`: TTS a prompt frames then b text-empty frames; audio_only a + b audio frames;
    text_only a + b text frames (audio rows the acoustic pad); ASR a audio frames (text row text-empty) then b text frames;
    then `pad` pad frames (semantic pad in row 1 for the audio tasks, text pad in row 0 for the text tasks)."""
    g = torch.Generator().manual_seed(seed)
    n = a + b
    seq = torch.randint(0, 2048, (9, n), generator=g)
    text = torch.randint(0, 1000, (n,), generator=g)
    if task == "TTS":
        seq[0, :a], seq[0, a:] = text[:a], T.TEXT_EMPTY
    elif task == "audio_only":
        seq[0] = T.TEXT_EMPTY
    elif task == "text_only":
        seq[0], seq[1:] = text, T.ACOUSTIC_PAD
    else:
        seq[0, :a], seq[0, a:], seq[1:, a:] = T.TEXT_EMPTY, text[a:], T.ACOUSTIC_PAD
    if pad:
        tail = torch.randint(0, 2048, (9, pad), generator=g)
        if task in ("audio_only", "TTS"):
            tail[1] = T.SEMANTIC_PAD
            tail[0] = T.TEXT_EMPTY if task == "audio_only" else 0
        else:
            tail[0] = T.TEXT_PAD
            tail[1:] = T.ACOUSTIC_PAD
        seq = torch.cat([seq, tail], 1)
    return seq


# (name, task, a, b, pad, seed, lengths or None)
ITEMS = [
    ("tts0", "TTS", 5, 8, 2, 11, None),
    ("tts1", "TTS", 9, 4, 0, 12, None),
    ("tts_open0", "TTS", 5, 8, 0, 13, (3, 20)),
    ("tts_open1", "TTS", 7, 6, 1, 14, (-2, 12)),
    ("audio0", "audio_only", 10, 4, 3, 21, None),
    ("audio1", "audio_only", 7, 8, 0, 22, None),
    ("text0", "text_only", 6, 6, 2, 31, None),
    ("text1", "text_only", 9, 4, 0, 32, None),
    ("asr0", "ASR", 6, 14, 2, 41, None),
    ("asr1", "ASR", 5, 15, 0, 42, None),
    ("asr2", "ASR", 7, 16, 1, 43, None),
    ("asr3", "ASR", 4, 14, 0, 44, None),
]


def run_reference(RefImp, m, task: str, seq: torch.Tensor, use_sampling: bool, tk: int) -> torch.Tensor:
    """the reference InferenceImp on one item -> its generated frames [G', 9] (TTS: rebuilt from its codes is not
    possible, so TTS returns the codes [8, G' - 1] instead)"""
    imp = RefImp(None, m, "sampling", 0.7, tk, 0.8, tk, task)
    imp.use_sampling = use_sampling        # instance attribute; the class hard-codes True (:162)
    with torch.no_grad():
        if task == "TTS":
            return imp(seq.clone(), torch.ones(seq.shape))
        try:
            imp(seq.clone(), torch.ones(seq.shape))
        except UnboundLocalError as e:
            tb = e.__traceback__
            while tb.tb_next is not None:
                tb = tb.tb_next
            line = traceback.extract_tb(tb)[-1]
            assert "gt_audio" in line.line and line.lineno == 299, f"the reference raised at {line.lineno}: {line.line}"
            loc = tb.tb_frame.f_locals
            return T.reference_frames(loc["final_results"], loc["prefix"], int(loc["pre_gen_len"]))
        raise AssertionError(f"the reference's {task} branch returned: the fixture's extraction no longer applies")


def main():
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    RefImp, _ = load_reference_inference_imp()
    save = {"stop_gain": np.array(STOP_GAIN), "stop_heads": np.array(STOP_HEADS), "context": np.array(CFG.context),
            "weights_sha256": np.array(weights_digest(task_weights())), "items": np.array([it[0] for it in ITEMS])}
    for name, task, a, b, pad, seed, lengths in ITEMS:
        seq = task_sequence(task, a, b, pad, seed)
        save[f"{name}_seq"] = seq.numpy()
        save[f"{name}_task"] = np.array(task)
        save[f"{name}_lengths"] = np.array(lengths if lengths is not None else (), dtype=np.int64)
    for dtype, tag in ((torch.float32, "f32"), (torch.bfloat16, "bf16")):
        w = task_weights()
        m = reference_gpt(w, CFG, dtype)
        m.load_state_dict(w, strict=True)
        m = m.to(dtype)
        wd = task_weights(dtype)
        for mode, use_sampling, tk in MODES:
            for name, task, a, b, pad, seed, lengths in ITEMS:
                seq = torch.from_numpy(save[f"{name}_seq"])
                with torch.no_grad():
                    mine = T.inference_imp(task, wd, CFG, seq.clone(), use_sampling, lengths=lengths)
                if lengths is None:
                    ref = run_reference(RefImp, m, task, seq, use_sampling, tk)
                    got = mine["codes"] if task == "TTS" else mine["frames"]
                    assert torch.equal(ref.cpu(), got), f"oracle != reference: {name} {tag} {mode}"
                k = f"{name}_{tag}_{mode}"
                save[f"{k}_frames"] = mine["frames"].numpy()
                save[f"{k}_margins"] = mine["margins"].numpy()
                save[f"{k}_stopped"] = np.array(mine["stopped"])
                save[f"{k}_window"] = np.array([mine["P"], mine["minlen"], mine["maxlen"]], dtype=np.int64)
                print(f"{name:10s} {tag} {mode:6s} P={mine['P']:2d} window=[{mine['minlen']}, {mine['maxlen']}] "
                      f"frames={mine['frames'].shape[0]:2d} stopped={mine['stopped']} "
                      f"min margin {float(mine['margins'].min()) if mine['margins'].numel() else float('nan'):.4f}"
                      f"{'' if lengths else ' == reference'}")
    os.makedirs(GOLDEN, exist_ok=True)
    np.savez_compressed(os.path.join(GOLDEN, "lm_tasks.npz"), **save)
    print("wrote", os.path.join(GOLDEN, "lm_tasks.npz"))


if __name__ == "__main__":
    sys.dont_write_bytecode = True
    main()
