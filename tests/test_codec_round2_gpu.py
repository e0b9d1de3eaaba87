"""GPU parity tests added in round 2 (-m gpu): the codec at BASELINE cfg 2's batch against the CPU oracle, index
equality wherever the float64 decision margin allows it (no blanket mismatch allowance), MimiTokenizer / MimiCodecBTK
through the kernels, per-stream reset / hold / state swap, and the batched frame scheduler."""
import os

import numpy as np
import pytest
import torch

from oracle import mimi_oracle as O
from oracle import mimi_spec as S

pytestmark = pytest.mark.gpu

from rstnet_b200.codec import MimiCodec, MimiCodecBTK, MimiTokenizer

DEV = "cuda"
MARGIN = 1e-4          # SURVEY.md H1: below this relative top-1/top-2 distance margin an index may flip under fp32 reordering


def _maxdiff(a, b):
    return (a.float().cpu() - b.float().cpu()).abs().max().item()


@pytest.fixture(scope="module")
def codec(official_weights):
    m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    m.load_state_dict(official_weights, strict=True)
    return m.to(DEV).eval()


def _oracle_stream(w, x, frames):
    """oracle streaming encode + decode (of its own codes), with the per-frame decision margins [B, frames]"""
    B = x.shape[0]
    sc = O.StreamingCodec(w, B)
    codes, wavs, margins = [], [], []
    with torch.no_grad():
        for i in range(frames):
            c = sc.encode(x[..., i * 1920:(i + 1) * 1920])
            margins.append(O.rvq_margins(sc.last_latent, w).min(dim=0).values.view(B, -1)[:, 0])
            codes.append(c)
            wavs.append(sc.decode(c))
    return torch.cat(codes, -1), torch.cat(wavs, -1), torch.stack(margins, 1)


@pytest.mark.parametrize("tc", [True, False])
def test_streaming_indices_equal_oracle_wherever_margins_allow(official_weights, codec, tc):
    """Tightened form of round 1's '<= 10 % of frames may differ': a frame may differ from the oracle only if its own
    float64 margin is below 1e-4 -- tensor-core (3xTF32) and FFMA paths alike."""
    x = S.synthetic_audio(6, 1920 * 8, seed=77)
    ref_codes, ref_wav, margins = _oracle_stream(official_weights, x, 8)
    codec.use_cuda_graphs, codec.streaming_tensor_cores = True, tc
    cs, ws = [], []
    with codec.streaming(6):
        for i in range(8):
            cs.append(codec.encode(x[..., i * 1920:(i + 1) * 1920].to(DEV)))
            ws.append(codec.decode(ref_codes[..., i:i + 1].to(DEV)))
    codes, wav = torch.cat(cs, -1).cpu(), torch.cat(ws, -1)
    bad = (codes != ref_codes).any(dim=1)                         # [B, frames]
    print(f"tc={tc}: {int(bad.sum())}/{bad.numel()} frames differ; smallest margin {float(margins.min()):.2e}")
    assert not bool((bad & (margins > MARGIN)).any())
    assert _maxdiff(wav, ref_wav) <= 1e-4 * max(1.0, float(ref_wav.abs().max()))


def test_cfg2_batch_256_vs_oracle(official_weights, codec):
    """BASELINE cfg 2's batch (256 independent streams, streaming, tensor cores, CUDA graphs) against the CPU oracle
    run at the same batch: 3 frames (frame 0 from silence-padded start, then two steady-state frames)."""
    B, frames = 256, 3
    x = S.synthetic_audio(B, 1920 * frames, seed=2024)
    ref_codes, ref_wav, margins = _oracle_stream(official_weights, x, frames)
    codec.use_cuda_graphs, codec.streaming_tensor_cores = True, True
    cs, ws = [], []
    with codec.streaming(B):
        for i in range(frames):
            cs.append(codec.encode(x[..., i * 1920:(i + 1) * 1920].to(DEV)))
            ws.append(codec.decode(ref_codes[..., i:i + 1].to(DEV)))
    codes, wav = torch.cat(cs, -1).cpu(), torch.cat(ws, -1)
    bad = (codes != ref_codes).any(dim=1)
    print(f"B=256: {int(bad.sum())}/{bad.numel()} frames differ from the oracle; {int((margins <= MARGIN).sum())} frames are near-ties; "
          f"wav max|d| {_maxdiff(wav, ref_wav):.2e}")
    assert not bool((bad & (margins > MARGIN)).any())
    assert _maxdiff(wav, ref_wav) <= 1e-4 * max(1.0, float(ref_wav.abs().max()))


def test_mimi_tokenizer_and_btk_layout(official_weights, codec):
    """MimiTokenizer.tokenize / detokenize (mimi_tokenizer.py:56-82: 2-D input, int16 storage, [8, T] layout) and the
    AudioCodec-tree [B, T, K] adapter, through the kernels."""
    tok = MimiTokenizer(codec, device=torch.device(DEV))
    x = S.synthetic_audio(1, 24000, seed=5)
    with torch.no_grad():
        ref_codes = O.encode(x, official_weights)
        z = O.encode_latent(x, official_weights)
        margins = O.rvq_margins(z, official_weights).min(dim=0).values
        ref_wav = O.decode(ref_codes, official_weights)
    codes = tok.tokenize(x[0], 24000)                              # wav [1, L]
    assert codes.dtype == torch.int16 and codes.shape == (8, 13) and not codes.is_cuda
    bad = (codes.long() != ref_codes[0]).any(dim=0)
    assert not bool((bad & (margins > MARGIN)).any())
    wav = tok.detokenize(ref_codes[0].to(torch.int16))
    assert wav.shape == (1, 24960) and not wav.is_cuda
    assert _maxdiff(wav, ref_wav[0]) <= 1e-4 * max(1.0, float(ref_wav.abs().max()))
    one_d = torch.arange(5)
    assert tok.tokenize(one_d) is one_d                            # already tokens (:62-63)
    assert tok.tokenize(torch.zeros(1, 0)) is None                 # empty clip (:66-67)
    with pytest.raises(NotImplementedError):
        tok.tokenize(x[0], 16000)
    assert tok.find_length(torch.zeros(8, 7)) == 7
    btk = MimiCodecBTK(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
    btk.load_state_dict(official_weights, strict=True)
    btk = btk.to(DEV).eval()
    xb = S.synthetic_audio(2, 5760, seed=6).to(DEV)
    c_btk, c_bkt = btk.encode(xb), codec.encode(xb)
    assert c_btk.shape == (2, 3, 8) and torch.equal(c_btk.transpose(1, 2), c_bkt)
    assert torch.equal(btk.decode(c_btk), codec.decode(c_bkt))


@pytest.mark.parametrize("tc", [True, False])
def test_per_stream_reset_hold_and_state_swap(codec, tc):
    """SURVEY.md §8f-1: (a) reset_streaming(streams=[i]) mid-run -> row i reproduces a fresh stream bit for bit, the
    other rows are undisturbed; (b) a held row (set_active_streams) keeps its exact state across a step it sits out;
    (c) get/set_streaming_state (modules/streaming.py:128-151) swap whole scopes."""
    B, frames = 5, 6
    x = S.synthetic_audio(B, 1920 * frames, seed=91).to(DEV)
    fr = lambda i: x[..., i * 1920:(i + 1) * 1920]
    codec.use_cuda_graphs, codec.streaming_tensor_cores = True, tc

    def run(step_inputs, hooks=None):
        outs = []
        with codec.streaming(B):
            for i, inp in enumerate(step_inputs):
                if hooks and i in hooks:
                    hooks[i]()
                c = codec.encode(inp)
                outs.append((c, codec.decode(c)))
        return outs

    base = run([fr(i) for i in range(frames)])
    # (a) row 1 restarts at step 3 and is fed frames 0, 1, 2 again
    inputs = [fr(i).clone() for i in range(frames)]
    for j, i in enumerate(range(3, 6)):
        inputs[i][1] = fr(j)[1]
    got = run(inputs, hooks={3: lambda: codec.reset_streaming(streams=[1])})
    others = [0, 2, 3, 4]
    for i in range(frames):
        assert torch.equal(got[i][0][others], base[i][0][others]) and torch.equal(got[i][1][others], base[i][1][others])
    for j, i in enumerate(range(3, 6)):
        assert torch.equal(got[i][0][1], base[j][0][1]) and torch.equal(got[i][1][1], base[j][1][1])
    # (b) rows 1 and 4 sit out step 2 (their input there is junk) and resume with their frame 2 at step 3
    inputs = [fr(0), fr(1), fr(2).clone(), fr(3).clone(), fr(4).clone()]
    inputs[2][[1, 4]] = 7.0
    inputs[3][[1, 4]] = fr(2)[[1, 4]]
    inputs[4][[1, 4]] = fr(3)[[1, 4]]
    mask = torch.ones(B, dtype=torch.int64); mask[[1, 4]] = 0
    got = run(inputs, hooks={2: lambda: codec.set_active_streams(mask), 3: lambda: codec.set_active_streams(None)})
    for i, src in ((3, 2), (4, 3)):
        assert torch.equal(got[i][0][[1, 4]], base[src][0][[1, 4]]) and torch.equal(got[i][1][[1, 4]], base[src][1][[1, 4]])
    for i in range(5):
        assert torch.equal(got[i][0][[0, 2, 3]], base[i][0][[0, 2, 3]]) and torch.equal(got[i][1][[0, 2, 3]], base[i][1][[0, 2, 3]])
    # (c) park a scope, run another one, resume the first
    codec.streaming_forever(B)
    c0 = codec.encode(fr(0))
    saved = codec.get_streaming_state()
    with codec.streaming(B):
        codec.encode(fr(3))
    codec.set_streaming_state(saved)
    c1 = codec.encode(fr(1))
    assert torch.equal(c0, base[0][0]) and torch.equal(c1, base[1][0])
    codec.set_streaming_state({"": None})
    assert not codec.is_streaming
    with pytest.raises(RuntimeError):
        codec.set_streaming_state({"x": None})


def test_frame_scheduler_with_duplex_engine(codec):
    """rstnet_b200.serve: sessions come and go in a live batch; a session's outputs do not depend on who else is in the
    batch, on its row, or on ticks it sat out (greedy decoding)."""
    from oracle import lm_oracle as L
    from rstnet_b200.lm import GPT, Config
    from rstnet_b200.serve import DuplexEngine, FrameScheduler
    cfg = L.SMALL
    lm = GPT(Config(block_size=cfg.block_size, n_layer=cfg.n_layer, n_embd=cfg.n_embd, n_head=cfg.n_head, head_size=cfg.head_size,
                    intermediate_size=cfg.intermediate_size, padded_vocab_size=cfg.padded_vocab_size, audio_card=cfg.audio_card,
                    n_q=cfg.n_q, dep_q=cfg.dep_q, codecformer_dim=cfg.codecformer_dim, codecformer_heads=cfg.codecformer_heads,
                    codecformer_layers=cfg.codecformer_layers, codecformer_dim_feedforward=cfg.codecformer_dim_feedforward,
                    context=cfg.context))
    lm.load_state_dict(L.synthetic_weights(cfg, seed=7, dtype=torch.float32, std=0.05), strict=True)
    lm = lm.to(DEV, torch.bfloat16).eval()
    codec.use_cuda_graphs, codec.streaming_tensor_cores = True, True
    audio = S.synthetic_audio(3, 1920 * 6, seed=55)
    fr = lambda s, i: audio[s, 0, i * 1920:(i + 1) * 1920]

    def session_alone(s):
        eng = DuplexEngine(codec, lm, 4, use_sampling=False)
        sch = FrameScheduler(eng, 4)
        sch.admit("x")
        out = []
        for i in range(6):
            sch.push("x", fr(s, i))
            out.append(sch.tick()["x"])
        return out

    alone = [session_alone(s) for s in range(3)]
    eng = DuplexEngine(codec, lm, 4, use_sampling=False)
    sch = FrameScheduler(eng, 4)
    sch.admit("A")
    got = {"A": [], "B": [], "C": []}
    nxt = {"A": 0, "B": 0, "C": 0}
    src = {"A": 0, "B": 1, "C": 2}
    for tick in range(9):
        if tick == 1:
            sch.admit("B")
        if tick == 3:
            sch.admit("C")
        for name in list(sch.sessions()):
            if name == "B" and tick == 4:
                continue                               # B delivers nothing this tick: it is held
            if nxt[name] < 6:
                sch.push(name, fr(src[name], nxt[name]))
                nxt[name] += 1
        for name, o in sch.tick().items():
            got[name].append(o)
        if tick == 6:
            sch.release("A")
    for name in ("A", "B", "C"):
        ref = alone[src[name]]
        assert len(got[name]) == 6, (name, len(got[name]))
        for (t_a, p_a), (t_b, p_b) in zip(got[name], ref):
            assert torch.equal(t_a, t_b) and torch.equal(p_a, p_b), name
    assert len(eng.latencies_ms) == 9 and sch.free_rows() == 2
    lm.streaming_forever(1); lm._state = None
    codec._stream_state = None


def test_offline_tokenization_and_batch_tensor_core_path(official_weights, codec, tmp_path):
    """rstnet_b200.offline (offline_codec_tokenization.py / inference.py drivers): equal-length clips are batched, the dict
    `utt -> int16 [8, T]` equals per-clip MimiTokenizer.tokenize and survives torch.save; a batch of >= 96 clips runs the
    non-streaming tensor-core path and must agree with the oracle wherever the margins allow; wav directory round trip."""
    from rstnet_b200 import offline
    tok = MimiTokenizer(codec, device=torch.device(DEV))
    lens = [4000, 9600, 9600, 1920, 9600, 5000]
    clips = {f"utt{i}": S.synthetic_audio(1, L, seed=300 + i)[0, 0] for i, L in enumerate(lens)}
    toks = offline.tokenize_utterances(codec, clips.items(), batch_size=2)
    assert set(toks) == set(clips)
    for utt, wav in clips.items():
        ref = tok.tokenize(wav[None], 24000)
        assert toks[utt].dtype == torch.int16 and torch.equal(toks[utt], ref), utt
    path = os.path.join(tmp_path, "codes.pt")
    offline.save_tokens(toks, path)
    back = torch.load(path)
    assert all(torch.equal(back[k], toks[k]) for k in toks)
    # a 128-clip batch: tensor-core batch plan vs the oracle
    B, L = 128, 1920 * 3
    x = S.synthetic_audio(B, L, seed=555)
    with torch.no_grad():
        ref_codes = O.encode(x, official_weights)
        margins = O.rvq_margins(O.encode_latent(x, official_weights), official_weights).min(dim=0).values.view(B, -1)
        ref_wav = O.decode(ref_codes, official_weights)
    codes = codec.encode(x.to(DEV))
    assert any(k[0] == "enc" and k[3] for k in codec._engine._plans), "the batch should have taken the tensor-core plan"
    bad = (codes.cpu() != ref_codes).any(dim=1)
    assert not bool((bad & (margins > MARGIN)).any())
    wav = codec.decode(ref_codes.to(DEV))
    assert _maxdiff(wav, ref_wav) <= 1e-4 * max(1.0, float(ref_wav.abs().max()))
    # wav directory round trip (inference.py)
    src, dst = os.path.join(tmp_path, "in"), os.path.join(tmp_path, "out")
    os.makedirs(src)
    offline.write_wav(os.path.join(src, "a.wav"), 0.5 * clips["utt1"] / clips["utt1"].abs().max())
    assert offline.reconstruct_directory(codec, src, dst) == 1
    rec, sr = offline.read_wav(os.path.join(dst, "a.wav"))
    assert sr == 24000 and rec.numel() == 9600


def test_fused_rope_attention_streaming_equals_separate_launches(official_weights):
    """MimiCodec.fused_rope_attention (default on) only removes 16 launches per frame: codes and PCM of a streaming run
    are bit-identical with the knob off."""
    x = S.synthetic_audio(4, 1920 * 5, seed=77).to(DEV)
    res = []
    for fused in (True, False):
        m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
        m.load_state_dict(official_weights, strict=True)
        m = m.to(DEV).eval()
        m.fused_rope_attention = fused
        cs, ws = [], []
        with m.streaming(4):
            for i in range(5):
                c = m.encode(x[..., i * 1920:(i + 1) * 1920])
                cs.append(c)
                ws.append(m.decode(c))
        res.append((torch.cat(cs, -1), torch.cat(ws, -1)))
    assert torch.equal(res[0][0], res[1][0])
    assert torch.equal(res[0][1], res[1][1])


def test_elu_in_transform_equals_elu_copy(official_weights):
    """MimiCodec.elu_in_transform_max_channels (default 0): the resblock conv reading the raw tensor and applying ELU in the
    GEMM's operand transform gives bit-identical codes and PCM to the default (ELU'd copy written by the producer)."""
    x = S.synthetic_audio(3, 1920 * 4, seed=78).to(DEV)
    res = []
    for ch in (128, 0):
        m = MimiCodec(encoder_rates=[8, 6, 5, 4], codebook_size=2048, codebook_dim=256, rvq_layers=8)
        m.load_state_dict(official_weights, strict=True)
        m = m.to(DEV).eval()
        m.elu_in_transform_max_channels = ch
        cs, ws = [], []
        with m.streaming(3):
            for i in range(4):
                c = m.encode(x[..., i * 1920:(i + 1) * 1920])
                cs.append(c)
                ws.append(m.decode(c))
        res.append((torch.cat(cs, -1), torch.cat(ws, -1)))
    assert torch.equal(res[0][0], res[1][0])
    assert torch.equal(res[0][1], res[1][1])
