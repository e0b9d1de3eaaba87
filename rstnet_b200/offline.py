"""Offline codec tokenization and reconstruction drivers (SURVEY.md §8f-3 / §8f-4).

  * `tokenize_utterances` / `python -m rstnet_b200.offline tokenize`: the Mimi branch of
    MLLM_v2/egs/pretraining/local/offline_codec_tokenization.py (and tools/data_scripts/offline_tokenization.py): every
    utterance -> int16 codes [8, T] of its 24 kHz audio, collected in a dict `utt_id -> tensor` and written with
    `torch.save` -- the on-disk format the reference's data loader reads (tools/tokenizer/MimiCodec/mimi_tokenizer.py:44,72).  Unlike the reference
    (one clip per call) clips of EQUAL length are encoded as one batch (>= 96 of them: on the tensor cores); clips are
    never padded to a common length, because the codec's convs zero-pad each LAYER's input at the end of a clip
    (modules/conv.py:245-254), so audio padding would change a clip's last frame.
  * `tokenize_corpus` / `tokenize --capacity N`: the same output through MimiCodec.encode_many -- clips of every length
    in one continuous batch of N rows on the streaming tensor-core path, equal to the per-clip result wherever the RVQ
    decision margin exceeds fp32 rounding (bit for bit on the fp32 CUDA-core path); without --capacity, tokenize stays
    pinned bit for bit to MimiTokenizer.tokenize.
  * `reconstruct_directory` / `python -m rstnet_b200.offline reconstruct`: AudioCodec/MimiCodec/inference.py:111-148 -- every
    wav of a directory through encode -> decode, written under the same name at 24 kHz.  `reconstruct_corpus` /
    `reconstruct --capacity N`: the same through encode_many -> decode_many.
  * `score` / `python -m rstnet_b200.offline score`: infer_no_streaming.py main() with --inference_mode teacher-force
    (:174-182) over a corpus (`torch.save`d dict utt_id -> {"seq": int64 [9, L], "mask": float [9, L]}) with
    InferenceImp.score_many: per-utterance losses / accuracies to a json file, and one json line with the mean
    loss_audio / 8, perplexity_audio = exp(that mean) and the mean text loss.  `score --model moshi` scores a Moshi
    fine-tune (the LMModel of rstnet_b200.moshi) as the reference trainer's validate_model does, with moshi.score_many over
    [n_q + 1, L] seq / mask items.
  * `synthesize` / `python -m rstnet_b200.offline synthesize`: the TTS loop of infer_no_streaming.py main() (:119-143) over a
    whole corpus (`torch.save`d dict utt_id -> int64 [9, L]) with InferenceImp.generate_many: utterances of any prompt and
    generation length decode together, a finished row taking the next utterance.  Writes utt_id -> int16 codes [8, T] and,
    with a codec, one 24 kHz 16-bit wav per utterance (Mimi decode of equal-length groups, as main()'s detokenize).
    `synthesize_stream` / `synthesize --stream`: the same codes through InferenceImp.stream_many, each wav decoded frame by
    frame during generation and written when its utterance completes.
  * `continue --model moshi` / `continue_corpus`: generation from a Moshi fine-tune over recorded dialogues (`torch.save`d
    dict utt_id -> int64 [n_q + 1, L], aligned): each prompted with its first --prompt-frames frames, then fed its
    recorded user channel, with moshi.generate_many; writes utt_id -> int64 [dep_q + 1, L - P] and, with a codec, the
    wavs of Moshi's audio channel through MimiCodec.decode_many.  --force audio takes Moshi's recorded audio at every
    frame and samples its text (row 0 of each output: a time-aligned transcript as token ids); --force text the reverse.

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
from typing import Dict, Iterable, Optional, Tuple

import numpy as np
import torch

from .audio import Resample
from .codec import MimiCodec
from .lm import kv_pages_for_budget


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


def _clips_24k(codec: MimiCodec, items: Iterable[Tuple], resamplers: Dict[int, Resample]):
    """(utt_id, 24 kHz wav [L] on the host) of every non-empty item; other rates through Resample(sr, 24000), one clip at a time."""
    for item in items:
        utt, wav = item[0], item[1]
        sr = int(item[2]) if len(item) > 2 else codec.sample_rate
        w = _as_row(wav)
        if not w.numel():
            continue
        if sr != codec.sample_rate:
            if sr not in resamplers:
                resamplers[sr] = Resample(sr, codec.sample_rate)
            w = resamplers[sr](w.to(codec.device)).cpu()
        yield utt, w


@torch.no_grad()
def tokenize_corpus(codec: MimiCodec, items: Iterable[Tuple], capacity: int = 128) -> Dict[str, torch.Tensor]:
    """`tokenize_utterances`' items and output ({utt_id: int16 [n_q, ceil(L24 / 1920)]}, empty clips skipped) through
    MimiCodec.encode_many: up to `capacity` clips of any lengths encode together, a finished clip's row taking the next."""
    clips = _clips_24k(codec, items, {})
    return {utt: codes.to(torch.int16) for utt, codes in codec.encode_many(clips, capacity)}


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
def reconstruct_corpus(codec: MimiCodec, src: str, dst: str, capacity: int = 128) -> int:
    """reconstruct_directory through encode_many -> decode_many: up to `capacity` files of any lengths in flight."""
    os.makedirs(dst, exist_ok=True)
    names = sorted(n for n in os.listdir(src) if n.lower().endswith(".wav"))
    lengths: Dict[str, int] = {}
    resamplers: Dict[int, Resample] = {}

    def clips():
        for name in names:
            wav, sr = read_wav(os.path.join(src, name))
            if sr != codec.sample_rate and wav.numel():
                if sr not in resamplers:
                    resamplers[sr] = Resample(sr, codec.sample_rate)
                wav = resamplers[sr](wav.to(codec.device)).cpu()
            lengths[name] = wav.numel()
            yield name, wav

    n = 0
    for name, rec in codec.decode_many(codec.encode_many(clips(), capacity), capacity):
        rec = rec[: lengths.pop(name)]
        if rec.numel() and float(rec.abs().max()) > 0.99:
            print(f"Clipping!! {name}: max scale {float(rec.abs().max()):.3f}", file=sys.stderr)
        write_wav(os.path.join(dst, name), rec, codec.sample_rate)
        n += 1
    return n


@torch.no_grad()
def synthesize(imp, corpus: Dict[str, torch.Tensor], capacity: int = 32, seeds=None,
               kv_gb: Optional[float] = None, n_samples: int = 1, all_samples: bool = False,
               lengths: Optional[Tuple[int, int]] = None) -> Dict[str, torch.Tensor]:
    """{utt_id: int16 [8, T]} for every utterance of `corpus` ({utt_id: int64 [9, L]}), through imp.generate_many.
    kv_gb: the KV cache's budget in GiB (a pool of floor(kv_gb * 2^30 / kv_page_bytes) pages); None: a whole ring per row.
    n_samples N > 1: best-of-N, the codes of each utterance's candidate with the highest mean audio log-probability per
    frame; all_samples also returns candidate i's codes as `<utt_id>_s<i>`.
    imp.task_name other than TTS: audio_only gives each item's prompt audio and continuation as one clip
    (infer.continuation_codes), int16 [8, P + G' - 1]; text_only and ASR the generated text token ids, int64 [G'].
    lengths: (min_frames, max_frames) replaces every item's window (generate_many's `lengths`)."""
    from .infer import continuation_codes
    corpus = {utt: torch.as_tensor(seq, dtype=torch.int64) for utt, seq in corpus.items()}
    kv_pages = None if kv_gb is None else kv_pages_for_budget(imp.model.config, kv_gb)
    lens = None if lengths is None else {utt: tuple(lengths) for utt in corpus}
    task = imp.task_name

    def result(utt, out):
        if task == "TTS":
            return out.to(torch.int16).cpu()
        if task == "audio_only":
            return continuation_codes(corpus[utt], out).to(torch.int16).cpu()
        return out[:, 0].cpu()

    out = {}
    for utt, res in imp.generate_many(iter(corpus.items()), capacity, seeds=seeds, kv_pages=kv_pages, n_samples=n_samples,
                                      lengths=lens):
        if n_samples == 1:
            out[utt] = result(utt, res)
            continue
        out[utt] = result(utt, res[0].codes)
        if all_samples:
            for c in sorted(res, key=lambda c: c.index):
                out[f"{utt}_s{c.index}"] = result(utt, c.codes)
    return out


@torch.no_grad()
def synthesize_stream(imp, codec: MimiCodec, corpus: Dict[str, torch.Tensor], dst: str, capacity: int = 32, seeds=None,
                      kv_gb: Optional[float] = None, lengths: Optional[Tuple[int, int]] = None) -> Dict[str, torch.Tensor]:
    """`synthesize` through imp.stream_many: the same {utt_id: int16 [8, T]}, and each utterance's `<utt_id>_sample.wav`
    (24 kHz 16-bit, as write_codes_wav; none for T = 0) written from its streamed chunks as soon as it completes."""
    os.makedirs(dst, exist_ok=True)
    items = ((utt, torch.as_tensor(seq, dtype=torch.int64)) for utt, seq in corpus.items())
    kv_pages = None if kv_gb is None else kv_pages_for_budget(imp.model.config, kv_gb)
    parts, out = defaultdict(list), {}
    lens = None if lengths is None else {utt: tuple(lengths) for utt in corpus}
    for ch in imp.stream_many(items, capacity, codec, seeds=seeds, kv_pages=kv_pages, lengths=lens):
        parts[ch.utt_id].append(ch.pcm)
        if ch.codes is not None:
            wav = torch.cat(parts.pop(ch.utt_id))
            if wav.numel():
                write_wav(os.path.join(dst, f"{ch.utt_id}_sample.wav"), wav, codec.sample_rate)
            out[ch.utt_id] = ch.codes.to(torch.int16)
    return out


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


def _positive_float(text: str) -> float:
    v = float(text)
    if not (v > 0 and np.isfinite(v)):
        raise argparse.ArgumentTypeError(f"must be a positive number (got {text})")
    return v


def _nonnegative_int(text: str) -> int:
    v = int(text)
    if v < 0:
        raise argparse.ArgumentTypeError(f"must be an integer >= 0 (got {text})")
    return v


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
    imp = InferenceImp(None, model, "sampling", args.temp_text, args.top_k_text, args.temp, args.top_k, args.task)
    if (args.min_frames is None) != (args.max_frames is None):
        raise SystemExit("--min-frames and --max-frames go together")
    lengths = None if args.min_frames is None else (args.min_frames, args.max_frames)
    if args.task in ("text_only", "ASR") and (args.stream or args.wav_dir):
        raise SystemExit(f"--task {args.task} writes text token ids: no --stream / --wav-dir")
    if args.task == "audio_only" and args.stream:
        raise SystemExit("--stream decodes the generated frames only; audio_only writes prompt + continuation: drop --stream")
    imp.use_sampling = args.use_sampling
    imp.top_p, imp.top_p_text = args.top_p, args.top_p_text
    if args.top_p or args.top_p_text:
        imp.sampling()   # validates a nucleus run's settings before the model runs
    corpus = torch.load(args.input, map_location="cpu")
    if args.all_samples and args.n_samples == 1:
        raise SystemExit("--all-samples needs --n-samples > 1")
    if args.stream:
        if args.n_samples != 1:
            raise SystemExit("--stream takes --n-samples 1: a streamed chunk cannot wait for the candidates' ranking")
        if not (args.wav_dir and args.codec_weights):
            raise SystemExit("--stream needs --wav-dir and --codec-weights")
        codec = _load_codec(argparse.Namespace(weights=args.codec_weights, config=args.codec_config, device=args.device))
        codes = synthesize_stream(imp, codec, corpus, args.wav_dir, args.capacity, kv_gb=args.kv_gb, lengths=lengths)
        save_tokens(codes, args.output_file)
        print(f"synthesized {len(codes)} utterances -> {args.output_file}, streamed their wavs -> {args.wav_dir}")
        return 0
    codes = synthesize(imp, corpus, args.capacity, kv_gb=args.kv_gb, n_samples=args.n_samples, all_samples=args.all_samples,
                       lengths=lengths)
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


def _load_moshi(config_path: str, checkpoint: str, device: str):
    """moshi.LMModel(**json) with the checkpoint's weights (a state_dict, or {'model': state_dict}; `module.` prefixes
    stripped), in bf16 on `device`."""
    import json
    from .moshi import LMModel
    m = LMModel(**json.load(open(config_path)))
    sd = torch.load(checkpoint, map_location="cpu")
    sd = sd["model"] if isinstance(sd, dict) and "model" in sd and isinstance(sd["model"], dict) else sd
    m.load_state_dict({k.split("module.")[-1] if k.startswith("module.") else k: v for k, v in sd.items()})
    return m.to(device, torch.bfloat16).eval()


def moshi_score_summary(metrics: Dict[str, dict], audio_weights=None) -> dict:
    """Corpus metrics of `score --model moshi`, pooled from the summed per-codebook sums: every scored token weighs the
    same, whatever its utterance (loss_k = sum of mask * nll over the corpus / count of non-zero mask entries).  The
    reference trainer's reporter instead averages the per-batch values, so its numbers depend on the batching."""
    from .lm import combine_sums
    from .moshi import AUDIO_WEIGHTS
    aw = AUDIO_WEIGHTS if audio_weights is None else audio_weights
    sa = sum((torch.tensor(m["sums_audio"], dtype=torch.float64) for m in metrics.values()), torch.zeros(len(aw), 5, dtype=torch.float64))
    st = sum((torch.tensor(m["sums_text"], dtype=torch.float64) for m in metrics.values()), torch.zeros(1, 5, dtype=torch.float64))
    a, t = combine_sums(sa, aw), combine_sums(st, [1])
    return {"utterances": len(metrics), "frames": sum(m["frames"] for m in metrics.values()), "loss_audio": float(a["loss"]),
            "loss_text": float(t["loss"]), "acc_audio": float(a["acc_all"]), "acc_text": float(t["acc_all"]),
            "acc_target_audio": float(a["acc_target"]), "acc_target_text": float(t["acc_target"])}


def _score_cli(args) -> int:
    import json
    from .infer import InferenceImp
    if args.model == "moshi":
        from .moshi import score_many
        model = _load_moshi(args.config, args.checkpoint, args.device)
        corpus = torch.load(args.input, map_location="cpu")
        items = ((utt, torch.as_tensor(d["seq"]), torch.as_tensor(d["mask"])) for utt, d in corpus.items())
        metrics = dict(score_many(model, items, args.capacity))
        with open(args.output_file, "w") as f:
            json.dump(metrics, f)
        print(json.dumps(moshi_score_summary(metrics)))
        return 0
    model = _load_gpt(args.config, args.checkpoint, args.device)
    imp = InferenceImp(None, model, "teacher-force", 0.7, 25, 0.8, 30, "TTS")
    corpus = torch.load(args.input, map_location="cpu")
    metrics = score(imp, corpus, args.capacity)
    with open(args.output_file, "w") as f:
        json.dump(metrics, f)
    print(json.dumps(score_summary(metrics)))
    return 0


@torch.no_grad()
def continue_corpus(gen, corpus: Dict[str, torch.Tensor], prompt_frames: int, capacity: int, kv_pages=None,
                    seed: int = 0, force: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """{utt: int64 [dep_q + 1, L - P]} of moshi.generate_many over `corpus` ({utt: int64 [K, L]} aligned dialogue codes),
    every item prompted with its first P = prompt_frames frames and seeded with `seed`.  force 'text': every item's text
    channel is taken from the recording at every frame and its audio sampled (re-voicing); 'audio': its audio codebooks
    1..dep_q are taken and its text sampled, so row 0 of the output is a time-aligned transcript (as token ids)."""
    from .moshi import generate_many
    items = [(utt, torch.as_tensor(seq), prompt_frames) for utt, seq in corpus.items()]
    seeds = {utt: seed for utt, _, _ in items}
    masks = None
    if force is not None:
        if force not in ("text", "audio"):
            raise ValueError(f"force is 'text' or 'audio' (got {force!r})")
        dq = gen.lm_model.dep_q
        masks = {}
        for utt, seq, _ in items:
            m = torch.zeros(dq + 1, seq.shape[1], dtype=torch.bool)
            m[slice(0, 1) if force == "text" else slice(1, dq + 1)] = True
            masks[utt] = m
    return dict(generate_many(gen, items, capacity, seeds=seeds, kv_pages=kv_pages, force=masks))


def continuation_wavs(codec: MimiCodec, out: Dict[str, torch.Tensor], prompt_frames: int, max_delay: int, dep_q: int,
                      capacity: int = 64):
    """{utt: float32 wav} of Moshi's audio channel in `continue_corpus`'s outputs through MimiCodec.decode_many: the
    columns that carry an aligned frame (step >= max_delay), audio codebooks 1..dep_q clamped to the codebook."""
    j0 = max(0, max_delay - prompt_frames)
    items = [(u, o[1:dep_q + 1, j0:].clamp(0, codec.codebook_size - 1)) for u, o in out.items() if o.shape[1] > j0]
    return dict(codec.decode_many(items, capacity))


def _continue_cli(args) -> int:
    from .lm import kv_pages_for_budget
    from .moshi import LMGen
    model = _load_moshi(args.config, args.checkpoint, args.device)
    gen = LMGen(model, use_sampling=args.use_sampling, temp=args.temp, temp_text=args.temp_text, top_k=args.top_k,
                top_k_text=args.top_k_text)
    corpus = torch.load(args.input, map_location="cpu")
    kv_pages = None if args.kv_gb is None else kv_pages_for_budget(model.config, args.kv_gb)
    out = continue_corpus(gen, corpus, args.prompt_frames, args.capacity, kv_pages=kv_pages, seed=args.seed, force=args.force)
    torch.save(out, args.output_file)
    print(f"continued {len(out)} dialogues -> {args.output_file}")
    if args.wav_dir:
        if not args.codec_checkpoint:
            raise SystemExit("--wav-dir needs --codec-checkpoint")
        codec = _load_codec(argparse.Namespace(weights=args.codec_checkpoint, config=args.codec_config, device=args.device))
        os.makedirs(args.wav_dir, exist_ok=True)
        wavs = continuation_wavs(codec, out, args.prompt_frames, max(model.delays), model.dep_q)
        for utt, w in wavs.items():
            write_wav(os.path.join(args.wav_dir, f"{utt}_sample.wav"), w, codec.sample_rate)
        print(f"wrote {len(wavs)} wavs -> {args.wav_dir}")
    return 0


def _load_codec(args) -> MimiCodec:
    import json
    cfg = json.load(open(args.config)) if args.config else dict(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m = MimiCodec(**cfg)
    sd = torch.load(args.weights, map_location="cpu")
    m.load_state_dict(sd.get("codec_model", sd), strict=False)
    return m.to(args.device).eval()


def pair_files(ref_dir: str, deg_dir: str):
    """[(name, ref_path, deg_path)] for every *.wav of deg_dir, paired by basename with ref_dir (compute_ms_stft_loss.py:108,
    123); a degraded file without a reference is an error that names the files."""
    names = sorted(n for n in os.listdir(deg_dir) if n.endswith(".wav"))
    if not names:
        raise FileNotFoundError(f"found no wavs in {deg_dir}")
    missing = [n for n in names if not os.path.isfile(os.path.join(ref_dir, n))]
    if missing:
        shown = ", ".join(missing[:10]) + (f" and {len(missing) - 10} more" if len(missing) > 10 else "")
        raise FileNotFoundError(f"{len(missing)} degraded file(s) of {deg_dir} have no reference in {ref_dir}: {shown}")
    return [(n, os.path.join(ref_dir, n), os.path.join(deg_dir, n)) for n in names]


def _evaluate_cli(args) -> int:
    import json
    from . import metrics as M
    pairs = pair_files(args.ref_dir, args.deg_dir)

    def items():
        for name, rp, dp in pairs:
            ref, rsr = read_wav(rp)
            deg, dsr = read_wav(dp)
            yield name, ref, rsr, deg, dsr
    capacity = max(1, int(round(args.capacity_seconds * args.sample_rate)))
    per_clip = dict(M.evaluate_pairs(items(), args.sample_rate, capacity, device=args.device))
    summary = M.corpus_summary(per_clip)
    with open(args.output_file, "w") as f:
        json.dump({"sample_rate": args.sample_rate, "summary": summary, "clips": per_clip}, f, indent=1)
    print(f"MS-STFT-Loss: {summary['ms_stft']}")
    print(f"SI-SNR: {summary['sisnr']}")
    if summary["stft_skipped"] or summary["sisnr_skipped"]:
        print(f"skipped: {summary['stft_skipped']} clip(s) too short for the STFT loss, {summary['sisnr_skipped']} without an "
              "SI-SNR (empty or constant reference)", file=sys.stderr)
    return 0


def main(argv=None) -> int:
    args = build_parser().parse_args(argv)
    if args.cmd == "evaluate":
        return _evaluate_cli(args)
    if args.cmd == "synthesize":
        return _synthesize_cli(args)
    if args.cmd == "score":
        return _score_cli(args)
    if args.cmd == "continue":
        return _continue_cli(args)
    codec = _load_codec(args)
    if args.cmd == "tokenize":
        def items():
            for line in open(args.wav_scp):
                utt, path = line.strip().split(None, 1)
                wav, sr = read_wav(path)
                yield utt, wav, sr
        if args.capacity is None:
            toks = tokenize_utterances(codec, items(), args.batch_size)
        else:
            toks = tokenize_corpus(codec, items(), args.capacity)
        save_tokens(toks, args.output_file)
        print(f"tokenized {len(toks)} utterances -> {args.output_file}")
    else:
        if args.capacity is None:
            n = reconstruct_directory(codec, args.input, args.output)
        else:
            n = reconstruct_corpus(codec, args.input, args.output, args.capacity)
        print(f"reconstructed {n} files -> {args.output}")
    return 0


def build_parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    for name in ("tokenize", "reconstruct"):
        p = sub.add_parser(name)
        p.add_argument("--weights", required=True, help="checkpoint (state_dict, or {'codec_model': state_dict})")
        p.add_argument("--config", default=None, help="json with the MimiCodec constructor arguments")
        p.add_argument("--device", default="cuda")
        p.add_argument("--capacity", type=int, default=None,
                       help="clips in flight at once: encode (and decode) every length in one continuous batch on the "
                            "streaming tensor-core path; without it, equal-length groups as MimiTokenizer does clip by clip")
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
    p.add_argument("--kv-gb", type=_positive_float, default=None,
                   help="KV cache budget in GiB: each utterance holds pages for only the positions it writes and waits for "
                        "pages when the budget is spent (default: a whole context ring per row)")
    p.add_argument("--use-sampling", action=argparse.BooleanOptionalAction, default=True,
                   help="sample (the reference hard-codes this); --no-use-sampling decodes by argmax")
    p.add_argument("--temp", type=float, default=0.8)
    p.add_argument("--top-k", type=int, default=30)
    p.add_argument("--temp-text", type=float, default=0.7)
    p.add_argument("--top-k-text", type=int, default=25)
    p.add_argument("--top-p", type=float, default=0.0, help="nucleus sampling of the audio heads (0: off; takes precedence over --top-k)")
    p.add_argument("--top-p-text", type=float, default=0.0, help="nucleus sampling of the text head (0: off)")
    p.add_argument("--wav-dir", default=None, help="also write <utt_id>_sample.wav here (needs --codec-weights)")
    p.add_argument("--codec-weights", default=None)
    p.add_argument("--codec-config", default=None, help="json with the MimiCodec constructor arguments")
    p.add_argument("--stream", action="store_true",
                   help="with --wav-dir: decode each utterance's audio frame by frame while it generates "
                        "(InferenceImp.stream_many) and write its wav as it completes; the codes file is the same")
    p.add_argument("--n-samples", type=int, default=1,
                   help="best-of-N: sample N candidates of each utterance from one prompt prefill (sharing its KV pages) and "
                        "keep the one with the highest mean audio log-probability per frame")
    p.add_argument("--all-samples", action="store_true", help="with --n-samples: also write candidate i as <utt_id>_s<i>")
    p.add_argument("--task", choices=("TTS", "audio_only", "text_only", "ASR"), default="TTS",
                   help="the reference loop's task and layout; audio_only writes prompt + continuation codes, text_only and "
                        "ASR the generated text token ids (int64 [G'])")
    p.add_argument("--min-frames", type=int, default=None,
                   help="with --max-frames: every item's window (minlen): the stop rule applies from frame min + 1 on")
    p.add_argument("--max-frames", type=int, default=None, help="with --min-frames: at most this many generated frames")
    p.add_argument("--device", default="cuda")
    p = sub.add_parser("score", help="teacher-forced losses / audio perplexity of a corpus (infer_no_streaming.py teacher-force; "
                                     "--model moshi: the Moshi fine-tune trainer's validate_model)")
    p.add_argument("--input", required=True, help="torch.save'd dict utt_id -> {'seq': int64 [9, L], 'mask': float [9, L]} "
                                                  "([n_q + 1, L] with --model moshi)")
    p.add_argument("--model", choices=("gpt", "moshi"), default="gpt",
                   help="gpt: the speech-text GPT; moshi: the Moshi-style LMModel (--config holds its constructor kwargs)")
    p.add_argument("--config", required=True, help="json with the GPT Config fields (--model moshi: the LMModel kwargs)")
    p.add_argument("--checkpoint", required=True, help="training checkpoint ({'model': state_dict}; --model moshi also takes a "
                                                       "bare state_dict)")
    p.add_argument("--output-file", required=True, help="json file of per-utterance metrics")
    p.add_argument("--capacity", type=int, default=8, help="utterances packed into the same chunks (<= 256)")
    p.add_argument("--device", default="cuda")
    p = sub.add_parser("continue", help="continue recorded dialogues with a Moshi fine-tune: each prompted with its first "
                                        "--prompt-frames frames, then fed its recorded user channel (moshi.generate_many)")
    p.add_argument("--model", choices=("moshi",), required=True, help="the Moshi-style LMModel (--config: its kwargs)")
    p.add_argument("--config", required=True, help="json with the LMModel constructor kwargs")
    p.add_argument("--checkpoint", required=True, help="a state_dict or {'model': state_dict}")
    p.add_argument("--input", required=True, help="torch.save'd dict utt_id -> int64 [n_q + 1, L], aligned (text, Moshi "
                                                  "audio, user audio)")
    p.add_argument("--prompt-frames", type=_nonnegative_int, required=True, help="P: frames of each dialogue taken as the prompt (< L)")
    p.add_argument("--output-file", required=True, help="torch.save'd dict utt_id -> int64 [dep_q + 1, L - P]")
    p.add_argument("--capacity", type=int, default=32, help="dialogues generated together (<= 256)")
    p.add_argument("--kv-gb", type=_positive_float, default=None,
                   help="KV cache budget in GiB (paged; default: a whole context ring per row)")
    p.add_argument("--seed", type=int, default=0, help="every dialogue's random stream")
    p.add_argument("--force", choices=("text", "audio"), default=None,
                   help="take this channel of Moshi's side from the recording at every frame and sample only the other: "
                        "'audio' writes a time-aligned transcript (row 0, token ids), 'text' re-voices the recorded text")
    p.add_argument("--use-sampling", action=argparse.BooleanOptionalAction, default=True)
    p.add_argument("--temp", type=float, default=0.8)
    p.add_argument("--top-k", type=int, default=250)
    p.add_argument("--temp-text", type=float, default=0.7)
    p.add_argument("--top-k-text", type=int, default=25)
    p.add_argument("--wav-dir", default=None, help="also write <utt_id>_sample.wav of Moshi's audio (needs --codec-checkpoint)")
    p.add_argument("--codec-checkpoint", default=None)
    p.add_argument("--codec-config", default=None, help="json with the MimiCodec constructor arguments")
    p.add_argument("--device", default="cuda")
    p = sub.add_parser("evaluate", help="multi-resolution STFT loss and SI-SNR of degraded wavs against references "
                                        "(Evaluation/codec/compute_ms_stft_loss.py, compute_sisnr.py)")
    p.add_argument("--ref-dir", required=True, help="reference wavs")
    p.add_argument("--deg-dir", required=True, help="degraded wavs, paired with --ref-dir by file name")
    p.add_argument("--sample-rate", type=int, default=16000, help="both signals are resampled to this rate (default 16000)")
    p.add_argument("--capacity-seconds", type=_positive_float, default=600.0,
                   help="audio per launch at --sample-rate (a longer clip runs alone)")
    p.add_argument("--output-file", default="metrics.json", help="json: per-clip metrics, corpus means, skipped counts")
    p.add_argument("--device", default="cuda")
    return ap


if __name__ == "__main__":
    sys.exit(main())
