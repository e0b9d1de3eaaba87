"""Offline codec tokenization and reconstruction drivers (SURVEY.md §8f-3 / §8f-4).

  * `tokenize_utterances` / `python -m rstnet_b200.offline tokenize`: the Mimi branch of
    MLLM_v2/egs/pretraining/local/offline_codec_tokenization.py (and tools/data_scripts/offline_tokenization.py): every
    utterance -> int16 codes [8, T] of its 24 kHz audio, collected in a dict `utt_id -> tensor` and written with
    `torch.save` -- the on-disk format the reference's data loader reads (tools/tokenizer/MimiCodec/mimi_tokenizer.py:44,72).  Unlike the reference
    (one clip per call) clips of EQUAL length are encoded as one batch (>= 96 of them: on the tensor cores); clips are
    never padded to a common length, because the codec's convs zero-pad each LAYER's input at the end of a clip
    (modules/conv.py:245-254), so audio padding would change a clip's last frame.
  * `reconstruct_directory` / `python -m rstnet_b200.offline reconstruct`: AudioCodec/MimiCodec/inference.py:111-148 -- every
    wav of a directory through encode -> decode, written under the same name at 24 kHz.
  * `score` / `python -m rstnet_b200.offline score`: infer_no_streaming.py main() with --inference_mode teacher-force
    (:174-182) over a corpus (`torch.save`d dict utt_id -> {"seq": int64 [9, L], "mask": float [9, L]}) with
    InferenceImp.score_many: per-utterance losses / accuracies to a json file, and one json line with the mean
    loss_audio / 8, perplexity_audio = exp(that mean) and the mean text loss.
  * `synthesize` / `python -m rstnet_b200.offline synthesize`: the TTS loop of infer_no_streaming.py main() (:119-143) over a
    whole corpus (`torch.save`d dict utt_id -> int64 [9, L]) with InferenceImp.generate_many: utterances of any prompt and
    generation length decode together, a finished row taking the next utterance.  Writes utt_id -> int16 codes [8, T] and,
    with a codec, one 24 kHz 16-bit wav per utterance (Mimi decode of equal-length groups, as main()'s detokenize).

Audio at any integer sample rate is resampled to 24 kHz on the GPU the way the reference does it,
torchaudio.transforms.Resample(sr, 24000) with its defaults (mimi_tokenizer.py:40,67; inference.py:24-34 `convert_audio`:
mean over channels, then Resample), by rstnet_b200.audio.Resample: clips of one (rate, length) group in one launch.
24 kHz clips go straight to the codec, as before.  Wav files are read and written through scipy.io.wavfile (mono mix of
the channels; integer PCM scaled to [-1, 1]).
"""
from __future__ import annotations

import argparse
import os
import sys
from collections import defaultdict
from typing import Dict, Iterable, Tuple

import numpy as np
import torch

from .audio import Resample
from .codec import MimiCodec


def _as_row(wav: torch.Tensor) -> torch.Tensor:
    wav = torch.as_tensor(wav, dtype=torch.float32)
    if wav.dim() == 2:
        if wav.shape[0] != 1:
            raise ValueError(f"mono audio expected, got {tuple(wav.shape)}")
        wav = wav[0]
    if wav.dim() != 1:
        raise ValueError(f"expected [L] or [1, L] audio, got {tuple(wav.shape)}")
    return wav


@torch.no_grad()
def tokenize_utterances(codec: MimiCodec, items: Iterable[Tuple], batch_size: int = 256) -> Dict[str, torch.Tensor]:
    """{utt_id: int16 [n_q, ceil(L24 / 1920)]} -- identical to MimiTokenizer.tokenize on every clip.  An item is
    (utt_id, wav) for 24 kHz audio or (utt_id, wav, sample_rate); other rates are resampled to 24 kHz first
    (Resample(sample_rate, 24000), one launch per batch of equal rate and length)."""
    dev = codec.device
    by_len = defaultdict(list)
    for item in items:
        utt, wav = item[0], item[1]
        sr = int(item[2]) if len(item) > 2 else codec.sample_rate
        w = _as_row(wav)
        if w.numel():
            by_len[(sr, w.numel())].append((utt, w))
    out: Dict[str, torch.Tensor] = {}
    resamplers: Dict[int, Resample] = {}
    for (sr, L), group in by_len.items():
        if sr != codec.sample_rate and sr not in resamplers:
            resamplers[sr] = Resample(sr, codec.sample_rate)
        for i in range(0, len(group), batch_size):
            part = group[i:i + batch_size]
            x = torch.stack([w for _, w in part])[:, None].to(dev)            # [B, 1, L]
            if sr != codec.sample_rate:
                x = resamplers[sr](x)                                        # [B, 1, ceil(L * 24000 / sr)]
            codes = codec.encode(x).to(torch.int16).cpu()                    # [B, n_q, T]
            for (utt, _), c in zip(part, codes):
                out[utt] = c.clone()
    return out


def save_tokens(tokens: Dict[str, torch.Tensor], path: str) -> None:
    torch.save(tokens, path)


def read_wav(path: str) -> Tuple[torch.Tensor, int]:
    from scipy.io import wavfile
    sr, data = wavfile.read(path)
    if data.ndim == 2:
        data = data.mean(axis=1)
    if np.issubdtype(data.dtype, np.integer):
        data = data.astype(np.float32) / float(np.iinfo(data.dtype).max)
    return torch.from_numpy(np.ascontiguousarray(data, dtype=np.float32)), int(sr)


def write_wav(path: str, wav: torch.Tensor, sr: int = 24000) -> None:
    from scipy.io import wavfile
    w = wav.detach().cpu().float().clamp(-1.0, 1.0).numpy()
    wavfile.write(path, sr, (w * 32767.0).astype(np.int16))


@torch.no_grad()
def reconstruct_directory(codec: MimiCodec, src: str, dst: str) -> int:
    """inference.py:test_batch -- wav -> codes -> wav for every file of `src`."""
    os.makedirs(dst, exist_ok=True)
    n = 0
    for name in sorted(os.listdir(src)):
        if not name.lower().endswith(".wav"):
            continue
        wav, sr = read_wav(os.path.join(src, name))
        wav = wav.to(codec.device)
        if sr != codec.sample_rate:
            wav = Resample(sr, codec.sample_rate)(wav)                       # convert_audio (inference.py:24-34)
        codes = codec.encode(wav[None, None].to(codec.device))
        rec = codec.decode(codes)[0, 0, : wav.numel()]
        if float(rec.abs().max()) > 0.99:
            print(f"Clipping!! {name}: max scale {float(rec.abs().max()):.3f}", file=sys.stderr)   # inference.py:check_clipping2
        write_wav(os.path.join(dst, name), rec, codec.sample_rate)
        n += 1
    return n


@torch.no_grad()
def synthesize(imp, corpus: Dict[str, torch.Tensor], capacity: int = 32, seeds=None) -> Dict[str, torch.Tensor]:
    """{utt_id: int16 [8, T]} for every utterance of `corpus` ({utt_id: int64 [9, L]}), through imp.generate_many."""
    items = ((utt, torch.as_tensor(seq, dtype=torch.int64)) for utt, seq in corpus.items())
    return {utt: codes.to(torch.int16).cpu() for utt, codes in imp.generate_many(items, capacity, seeds=seeds)}


@torch.no_grad()
def write_codes_wav(codec: MimiCodec, codes: Dict[str, torch.Tensor], dst: str, batch_size: int = 64) -> int:
    """One `<utt_id>_sample.wav` per utterance (main()'s file name), 24 kHz 16-bit: codes of equal length decode as one batch."""
    os.makedirs(dst, exist_ok=True)
    by_len = defaultdict(list)
    for utt, c in codes.items():
        if c.shape[-1] > 0:
            by_len[c.shape[-1]].append(utt)
    for T, utts in by_len.items():
        for i in range(0, len(utts), batch_size):
            part = utts[i:i + batch_size]
            wav = codec.decode(torch.stack([codes[u] for u in part]).to(torch.int64))
            for u, w in zip(part, wav):
                write_wav(os.path.join(dst, f"{u}_sample.wav"), w[0], codec.sample_rate)
    return sum(len(u) for u in by_len.values())


def _load_gpt(config_path: str, checkpoint: str, device: str):
    """GPT(Config from json) with the checkpoint's ['model'] weights, `module.` prefixes stripped
    (utils/train_utils.py:resume_for_inference), in bf16 on `device`."""
    import json
    from .lm import GPT, Config
    m = GPT(Config(**json.load(open(config_path))))
    sd = torch.load(checkpoint, map_location="cpu")["model"]
    m.load_state_dict({k.split("module.")[-1] if k.startswith("module.") else k: v for k, v in sd.items()})
    return m.to(device, torch.bfloat16).eval()


def _synthesize_cli(args) -> int:
    from .infer import InferenceImp
    model = _load_gpt(args.config, args.checkpoint, args.device)
    imp = InferenceImp(None, model, "sampling", args.temp_text, args.top_k_text, args.temp, args.top_k, "TTS")
    imp.use_sampling = args.use_sampling
    corpus = torch.load(args.input, map_location="cpu")
    codes = synthesize(imp, corpus, args.capacity)
    save_tokens(codes, args.output_file)
    print(f"synthesized {len(codes)} utterances -> {args.output_file}")
    if args.wav_dir:
        if not args.codec_weights:
            raise SystemExit("--wav-dir needs --codec-weights")
        codec = _load_codec(argparse.Namespace(weights=args.codec_weights, config=args.codec_config, device=args.device))
        print(f"wrote {write_codes_wav(codec, codes, args.wav_dir)} wavs -> {args.wav_dir}")
    return 0


@torch.no_grad()
def score(imp, corpus: Dict[str, dict], capacity: int = 8) -> Dict[str, dict]:
    """{utt_id: metrics} of InferenceImp.score_many over `corpus` ({utt_id: {"seq": int64 [9, L], "mask": float [9, L]}})."""
    items = ((utt, torch.as_tensor(d["seq"]), torch.as_tensor(d["mask"])) for utt, d in corpus.items())
    return dict(imp.score_many(items, capacity))


def score_summary(metrics: Dict[str, dict]) -> dict:
    """main()'s teacher-force report (infer_no_streaming.py:174-182): perplexity_audio = exp(mean over utterances of
    loss_audio / 8); the mean text loss beside it."""
    import math
    n = len(metrics)
    la = sum(m["loss_audio"] for m in metrics.values()) / n if n else float("nan")
    lt = sum(m["loss_text"] for m in metrics.values()) / n if n else float("nan")
    return {"utterances": n, "loss_audio": la, "perplexity_audio": math.exp(la) if la == la else float("nan"), "loss_text": lt}


def _score_cli(args) -> int:
    import json
    from .infer import InferenceImp
    model = _load_gpt(args.config, args.checkpoint, args.device)
    imp = InferenceImp(None, model, "teacher-force", 0.7, 25, 0.8, 30, "TTS")
    corpus = torch.load(args.input, map_location="cpu")
    metrics = score(imp, corpus, args.capacity)
    with open(args.output_file, "w") as f:
        json.dump(metrics, f)
    print(json.dumps(score_summary(metrics)))
    return 0


def _load_codec(args) -> MimiCodec:
    import json
    cfg = json.load(open(args.config)) if args.config else dict(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m = MimiCodec(**cfg)
    sd = torch.load(args.weights, map_location="cpu")
    m.load_state_dict(sd.get("codec_model", sd), strict=False)
    return m.to(args.device).eval()


def main(argv=None) -> int:
    args = build_parser().parse_args(argv)
    if args.cmd == "synthesize":
        return _synthesize_cli(args)
    if args.cmd == "score":
        return _score_cli(args)
    codec = _load_codec(args)
    if args.cmd == "tokenize":
        def items():
            for line in open(args.wav_scp):
                utt, path = line.strip().split(None, 1)
                wav, sr = read_wav(path)
                yield utt, wav, sr
        toks = tokenize_utterances(codec, items(), args.batch_size)
        save_tokens(toks, args.output_file)
        print(f"tokenized {len(toks)} utterances -> {args.output_file}")
    else:
        print(f"reconstructed {reconstruct_directory(codec, args.input, args.output)} files -> {args.output}")
    return 0


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    for name in ("tokenize", "reconstruct"):
        p = sub.add_parser(name)
        p.add_argument("--weights", required=True, help="checkpoint (state_dict, or {'codec_model': state_dict})")
        p.add_argument("--config", default=None, help="json with the MimiCodec constructor arguments")
        p.add_argument("--device", default="cuda")
    sub.choices["tokenize"].add_argument("--wav-scp", required=True, help="kaldi wav.scp: <utt_id> <path>")
    sub.choices["tokenize"].add_argument("--output-file", required=True)
    sub.choices["tokenize"].add_argument("--batch-size", type=int, default=256)
    sub.choices["reconstruct"].add_argument("--input", required=True)
    sub.choices["reconstruct"].add_argument("--output", required=True)
    p = sub.add_parser("synthesize", help="TTS codes for a corpus of utterances (infer_no_streaming.py main())")
    p.add_argument("--input", required=True, help="torch.save'd dict utt_id -> int64 [9, L]")
    p.add_argument("--config", required=True, help="json with the GPT Config fields")
    p.add_argument("--checkpoint", required=True, help="training checkpoint ({'model': state_dict})")
    p.add_argument("--output-file", required=True, help="torch.save'd dict utt_id -> int16 [8, T]")
    p.add_argument("--capacity", type=int, default=32, help="utterances decoded together (<= 256)")
    p.add_argument("--use-sampling", action=argparse.BooleanOptionalAction, default=True,
                   help="sample (the reference hard-codes this); --no-use-sampling decodes by argmax")
    p.add_argument("--temp", type=float, default=0.8)
    p.add_argument("--top-k", type=int, default=30)
    p.add_argument("--temp-text", type=float, default=0.7)
    p.add_argument("--top-k-text", type=int, default=25)
    p.add_argument("--wav-dir", default=None, help="also write <utt_id>_sample.wav here (needs --codec-weights)")
    p.add_argument("--codec-weights", default=None)
    p.add_argument("--codec-config", default=None, help="json with the MimiCodec constructor arguments")
    p.add_argument("--device", default="cuda")
    p = sub.add_parser("score", help="teacher-forced losses / audio perplexity of a corpus (infer_no_streaming.py teacher-force)")
    p.add_argument("--input", required=True, help="torch.save'd dict utt_id -> {'seq': int64 [9, L], 'mask': float [9, L]}")
    p.add_argument("--config", required=True, help="json with the GPT Config fields")
    p.add_argument("--checkpoint", required=True, help="training checkpoint ({'model': state_dict})")
    p.add_argument("--output-file", required=True, help="json file of per-utterance metrics")
    p.add_argument("--capacity", type=int, default=8, help="utterances packed into the same chunks (<= 256)")
    p.add_argument("--device", default="cuda")
    return ap


if __name__ == "__main__":
    sys.exit(main())
