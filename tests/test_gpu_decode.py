"""GPU parity tests for the KV-cached decode path (SURVEY.md section 8 row a9): token ids bit-exact at temperature 0
against the CPU oracle and against the fixture produced by the unmodified reference's decode_stable."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _mk(name_or_dims, seed):
    import oracle.whisper_ref as W
    from stable_ts_b200.model import from_oracle
    from stable_ts_b200.tokenizer import get_tokenizer
    model = W.build_model(name_or_dims, seed=seed)
    gm = from_oracle(model)
    tk = get_tokenizer(gm, language="en", task="transcribe", synthetic=True)
    return W, model, gm, tk


def _mel(W, model, audio):
    return W.pad_or_trim(W.log_mel_spectrogram(audio, model.dims.n_mels, padding=480000 - len(audio)), 3000)


@pytest.mark.parametrize("name", ["mini_en", "mini_ml"])
def test_decode_matches_reference_fixture(name):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import stable_path as SP
    from oracle.whisper_ref.model import ModelDimensions
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    z = np.load(os.path.join(GOLD, f"{name}.npz"))
    W, model, gm, tk = _mk(ModelDimensions(*[int(v) for v in z["dims"]]), int(z["model_seed"]))
    audio = SP.synth_audio(int(z["n_samples"]), seed=1234)
    enc = gm.encode(gm.log_mel(audio.cuda()[None]))
    mask = torch.zeros(1501, dtype=torch.bool)
    mask[100:400] = True
    res, ex = decode_windows(gm, tk, enc, DecodingOptions(language="en", sample_len=24), ts_token_mask=mask)
    print(f"[{name}] tokens {res[0].tokens[:8]} avg_logprob {res[0].avg_logprob:.5f} (ref {float(z['decode_avg_logprob']):.5f}) "
          f"no_speech {res[0].no_speech_prob:.3e} (ref {float(z['decode_no_speech']):.3e})")
    assert res[0].tokens == z["decode_tokens"].tolist()
    assert abs(res[0].avg_logprob - float(z["decode_avg_logprob"])) < 1e-3
    assert abs(res[0].no_speech_prob - float(z["decode_no_speech"])) <= 2e-3 * float(z["decode_no_speech"])


@pytest.mark.parametrize("name", ["tiny", "base.en"])
def test_free_running_greedy_batch_matches_oracle(name):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import stable_path as SP
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    W, model, gm, tk = _mk(name, 4)
    audios = [SP.synth_audio(480000, seed=31), SP.synth_audio(250000, seed=32), SP.synth_audio(100000, seed=33)]
    batch = torch.zeros(3, 480000)
    for i, a in enumerate(audios):
        batch[i, : len(a)] = a
    enc = gm.encode(gm.log_mel(batch.cuda()))
    mask = torch.zeros(1501, dtype=torch.bool)
    mask[700:1501] = True
    opt = DecodingOptions(language="en", sample_len=40)
    res_g, _ = decode_windows(gm, tk, enc, opt, ts_token_mask=mask, use_graph=True)
    res_e, _ = decode_windows(gm, tk, enc, opt, ts_token_mask=mask, use_graph=False)
    for b, a in enumerate(audios):
        ref, _, ex = SP.decode_window(model, _mel(W, model, a), ts_token_mask=mask, language="en", sample_len=40)
        print(f"[{name}] window {b}: {len(ref.tokens)} tokens, avg_logprob {res_g[b].avg_logprob:.5f} vs {ref.avg_logprob:.5f}")
        assert res_g[b].tokens == ref.tokens, (res_g[b].tokens, ref.tokens)
        assert res_e[b].tokens == ref.tokens
        assert abs(res_g[b].avg_logprob - ref.avg_logprob) < 1e-3
        assert abs(res_g[b].no_speech_prob - ref.no_speech_prob) <= 2e-3 * ref.no_speech_prob + 1e-12


def test_forced_script_step_logits_and_argmax():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import stable_path as SP
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    W, model, gm, tk = _mk("tiny.en", 6)
    audio = SP.synth_audio(480000, seed=41)
    enc = gm.encode(gm.log_mel(audio.cuda()[None]))
    steps = 48
    script = SP.synth_token_script(steps, tk.eot, seed=5)
    ref, _, ex = SP.decode_window(model, _mel(W, model, audio), forced_tokens=script, return_step_logits=True, sample_len=steps)
    res, gx = decode_windows(gm, tk, enc, DecodingOptions(sample_len=steps), forced_tokens=torch.tensor(script)[:, None],
                             return_step_logits=True)
    worst = 0.0
    for i in range(steps):
        r = ex["step_logits"][i]
        g = gx["step_logits"][i][0].cpu()
        fin = r > -1e30                      # nan_to_num_ turns the filters' -inf into the lowest finite float
        assert torch.equal(fin, g > -1e30), f"mask mismatch at step {i}"
        worst = max(worst, ((g[fin] - r[fin]).abs().max() / r[fin].abs().max()).item())
    print(f"forced 48-step script: worst step-logit rel err {worst:.2e}")
    assert worst < 1e-3
    assert gx["step_argmax"][:, 0].tolist() == ex["step_argmax"]
    res2, gx2 = decode_windows(gm, tk, enc, DecodingOptions(sample_len=steps), forced_tokens=torch.tensor(script)[:, None])
    assert gx2["step_argmax"][:, 0].tolist() == ex["step_argmax"]          # CUDA-graph replay path


@pytest.mark.parametrize("name", ["mini_en", "mini_ml"])
def test_transcribe_window_matches_reference_driver_fixture(name):
    """decode -> segment slicing -> gap-padded word timestamps of the first window == what the UNMODIFIED
    transcribe_stable produced (tests/golden/*_transcribe.json, oracle/make_golden.py)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import json
    from oracle import stable_path as SP
    from oracle.whisper_ref.model import ModelDimensions
    from stable_ts_b200.decode import DecodingOptions
    from stable_ts_b200.transcribe import transcribe_windows
    z = np.load(os.path.join(GOLD, f"{name}.npz"))
    gold = json.load(open(os.path.join(GOLD, f"{name}_transcribe.json")))
    W, model, gm, tk = _mk(ModelDimensions(*[int(v) for v in z["dims"]]), int(z["model_seed"]))
    audio = SP.synth_audio(int(z["n_samples"]), seed=1234)
    segs, info = transcribe_windows(gm, tk, [audio], options=DecodingOptions(language="en", sample_len=40, max_initial_timestamp=None))
    segs = segs[0]
    assert [s["tokens"] for s in segs] == [s["tokens"] for s in gold["segments"]]
    worst = 0.0
    for s, g in zip(segs, gold["segments"]):
        assert len(s["words"]) == len(g["words"])
        assert abs(s["start"] - g["start"]) <= 0.0201 and abs(s["end"] - g["end"]) <= 0.0201
        for w, gw in zip(s["words"], g["words"]):
            assert w["tokens"] == gw["tokens"] and w["word"] == gw["word"]
            worst = max(worst, abs(w["start"] - gw["start"]), abs(w["end"] - gw["end"]))
            assert abs(w["probability"] - gw["probability"]) <= 2e-3 * gw["probability"] + 1e-12
    print(f"[{name}] transcribe window: {len(segs)} segments, worst word |dt| {worst:.3f}s")
    assert worst <= 0.0201


def test_decode_large_batch_uses_tensor_core_step_and_matches_gemv_step():
    """18 sequences = two 16-row groups of the batched-GEMV step (the second one ragged): same tokens as 3 sequences."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import stable_path as SP
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    W, model, gm, tk = _mk("tiny.en", 8)
    audios = torch.stack([SP.synth_audio(480000, seed=60 + i) for i in range(3)])
    big = audios.repeat(6, 1)                                  # 18 windows (3 distinct)
    opt = DecodingOptions(sample_len=20)
    r18, _ = decode_windows(gm, tk, gm.encode(gm.log_mel(big.cuda())), opt)
    r3, _ = decode_windows(gm, tk, gm.encode(gm.log_mel(audios.cuda())), opt)
    for b in range(18):
        assert r18[b].tokens == r3[b % 3].tokens
        assert abs(r18[b].avg_logprob - r3[b % 3].avg_logprob) < 1e-4


def test_decode_batch_above_64_takes_tcgen05_step():
    """B > 64 falls to the wgmma small-M GEMM step; must agree with the batched-GEMV step on the same windows."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import stable_path as SP
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    W, model, gm, tk = _mk("tiny.en", 8)
    audios = torch.stack([SP.synth_audio(160000, seed=80 + i) for i in range(2)])
    pad = torch.zeros(2, 480000)
    pad[:, :160000] = audios
    opt = DecodingOptions(sample_len=12)
    r66, _ = decode_windows(gm, tk, gm.encode(gm.log_mel(pad.repeat(33, 1).cuda())), opt)
    r2, _ = decode_windows(gm, tk, gm.encode(gm.log_mel(pad.cuda())), opt)
    for b in range(66):
        assert r66[b].tokens == r2[b % 2].tokens


def test_large_width_step_paths_agree():
    """large-v3 widths (d = 1280, 20 heads, 51866 tokens; 1 encoder + 2 decoder layers): the two decode-step linear
    routes -- mma.sync GEMV (B = 2) and the cluster split-K wgmma kernel (B = 20 and 50: BN = 32 / 64, K = 1280 and 5120,
    vocabulary projection) -- must produce the same step logits and tokens."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import stable_path as SP
    from oracle.whisper_ref.model import ModelDimensions
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    dims = ModelDimensions(n_mels=128, n_audio_ctx=1500, n_audio_state=1280, n_audio_head=20, n_audio_layer=1, n_vocab=51866,
                           n_text_ctx=448, n_text_state=1280, n_text_head=20, n_text_layer=2)
    W, model, gm, tk = _mk(dims, 17)
    audios = torch.stack([SP.synth_audio(480000, seed=90 + i) for i in range(2)])
    enc2 = gm.encode(gm.log_mel(audios.cuda()))
    steps = 5
    opt = DecodingOptions(sample_len=steps)
    r2, x2 = decode_windows(gm, tk, enc2, opt, return_step_logits=True)
    V = dims.n_vocab
    for rep in (10, 25):
        encb = gm.encode(gm.log_mel(audios.repeat(rep, 1).cuda()))
        rb, xb = decode_windows(gm, tk, encb, opt, return_step_logits=True)
        worst = 0.0
        for i in range(len(x2["step_logits"])):
            a = x2["step_logits"][i].float().cpu()
            b = xb["step_logits"][i].float().cpu()
            fin = a > -1e30
            for j in range(2 * rep):
                assert torch.equal(fin[j % 2], b[j] > -1e30)
                worst = max(worst, ((b[j][fin[j % 2]] - a[j % 2][fin[j % 2]]).abs().max() / a[j % 2][fin[j % 2]].abs().max()).item())
        print(f"B={2 * rep} vs B=2 step logits: worst rel diff {worst:.2e}")
        assert worst < 2e-5
        for j in range(2 * rep):
            assert rb[j].tokens == r2[j % 2].tokens
        rg, _ = decode_windows(gm, tk, encb, opt)                     # CUDA-graph replay of the same step
        for j in range(2 * rep):
            assert rg[j].tokens == r2[j % 2].tokens


def test_cross_attention_step_logits_match_float64():
    """The decode-step cross-attention (mma.sync over TMA-swizzled fp16 K / V tiles) at large-v3 widths (d = 1280, 20 heads,
    51866 tokens; 1 encoder + 2 decoder layers), behind the GEMV (B = 3) and the cluster (B = 42) linears, with a window whose
    tail is silence: step logits of a forced token script against the oracle's decode in float64, fed this library's own
    encoder output so that only the decode step is measured.  Then graph replay against eager stepping, and a free-running
    tiny.en decode against the CPU oracle."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import copy
    import torch.nn.functional as F
    from oracle import stable_path as SP
    from oracle.whisper_ref import model as WM
    from oracle.whisper_ref.model import ModelDimensions
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    dims = ModelDimensions(n_mels=128, n_audio_ctx=1500, n_audio_state=1280, n_audio_head=20, n_audio_layer=1, n_vocab=51866,
                           n_text_ctx=448, n_text_state=1280, n_text_head=20, n_text_layer=2)
    W, model, gm, tk = _mk(dims, 17)
    m64 = copy.deepcopy(model).double()
    audios = torch.stack([SP.synth_audio(480000, seed=90 + i) for i in range(3)])
    audios[2, 200000:] = 0                                    # a window whose tail is silence
    steps = 8
    script = SP.synth_token_script(steps, tk.eot, seed=11)
    opt = DecodingOptions(language="en", sample_len=steps)
    mel = torch.zeros(dims.n_mels, 3000)                      # (not read: the oracle is given the audio features)
    refs = []                                                 # (float64 encoder output of a window, its step logits)
    with pytest.MonkeyPatch.context() as mp:
        # the oracle's LayerNorm computes in fp32 (a guard for fp16 models); in the float64 model it keeps float64
        mp.setattr(WM.LayerNorm, "forward", lambda self, x: F.layer_norm(x, self.normalized_shape, self.weight, self.bias, self.eps))
        for rep in (1, 14):                                   # B = 3 (GEMV linears) and B = 42 (cluster linears)
            B = 3 * rep
            enc = gm.encode(gm.log_mel(audios.repeat(rep, 1).cuda()))
            _, x = decode_windows(gm, tk, enc, opt, forced_tokens=torch.tensor(script)[:, None].repeat(1, B),
                                  return_step_logits=True)
            feats = enc["f32"].view(B, dims.n_audio_ctx, -1).cpu().double()
            worst = 0.0
            for j in range(B):
                ref = next((r for a, r in refs if torch.equal(a, feats[j])), None)
                if ref is None:
                    _, _, ex = SP.decode_window(m64, mel, audio_features=feats[j:j + 1], forced_tokens=script,
                                                return_step_logits=True, sample_len=steps, language="en")
                    ref = ex["step_logits"]
                    refs.append((feats[j], ref))
                assert len(ref) == len(x["step_logits"]) == steps
                for r, g in zip(ref, x["step_logits"]):
                    r, g = r.double(), g[j].double().cpu()
                    fin = r > -1e30
                    assert torch.equal(fin, g > -1e30)
                    worst = max(worst, ((g[fin] - r[fin]).abs().max() / r[fin].abs().max()).item())
            print(f"B={B}: decode step vs float64 oracle, worst step-logit rel err {worst:.2e}")
            # measured on an NVIDIA H100 80GB HBM3 at 700 W: 9.70e-6 (B = 3) and 1.19e-5 (B = 42) with this kernel, 9.75e-6
            # and 1.19e-5 with the scalar-lane kernel it replaced; the bound is 1.25x the worst, rounded up
            assert worst < 2e-5
            r_eager, _ = decode_windows(gm, tk, enc, opt, use_graph=False)
            r_graph, _ = decode_windows(gm, tk, enc, opt)     # CUDA-graph replay of the same step
            for a, b in zip(r_eager, r_graph):
                assert a.tokens == b.tokens
    # against the CPU oracle (tiny.en, free-running greedy)
    W2, om, gm2, tk2 = _mk("tiny.en", 3)
    audio = SP.synth_audio(480000, seed=7)
    ref, _, _ = SP.decode_window(om, _mel(W2, om, audio), language="en", sample_len=16)
    res, _ = decode_windows(gm2, tk2, gm2.encode(gm2.log_mel(audio.cuda()[None])), DecodingOptions(language="en", sample_len=16))
    assert res[0].tokens == ref.tokens and abs(res[0].avg_logprob - ref.avg_logprob) < 1e-3

