"""The decode step at and beyond its route boundaries (``decode_step``, ``csrc/engine.cu``): B <= 16 runs the step linears as
the batched GEMV, 17..128 as the cluster split-K kernel, and B > 128 as the plain ``gemm_tc`` GEMM plus a standalone LayerNorm.
Users reach B > 128 through ``transcribe_batch(batch_windows > 128)`` and through the temperature fallback with ``best_of``.

Only a few distinct windows are encoded, and the cross K/V block, KV cache and step workspace are the model-owned buffers
that ``transcribe`` reuses, so the device memory stays at one batch's worth.  The batch is tiled from them with ``enc_select`` as window b % 5 and forced script
b % 3, so a row that read row b - 64 or b - 128 would meet a different window and fail.
"""
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

ROUTES = {"gemv_mma_kernel": "GEMV", "decode_linear_kernel": "cluster", "gemm_tc_kernel": "GEMM"}


def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _mk(name_or_dims, seed):
    import oracle.whisper_ref as W
    from stable_ts_b200.model import from_oracle
    from stable_ts_b200.tokenizer import get_tokenizer
    model = W.build_model(name_or_dims, seed=seed)
    gm = from_oracle(model)
    tk = get_tokenizer(gm, language="en", task="transcribe", synthetic=True)
    return W, model, gm, tk


def _report(name, t0):
    print(f"{name}: {time.time() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def _step_route(gm, tk, enc, opt, ckv):
    """the step-linear kernels two eager decode steps launch (the cross K/V block is given, so no encoder GEMM runs)"""
    from stable_ts_b200.decode import decode_windows
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        decode_windows(gm, tk, enc, opt, ckv=ckv, use_graph=False)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    return {r for k, r in ROUTES.items() if any(k in n for n in names)}


def test_step_logits_across_the_route_boundaries_match_float64():
    """large-v3 widths (d = 1280, 20 heads, 51866 tokens; 1 encoder + 2 decoder layers) at B = 16 / 17 / 128 / 129 / 260:
    step logits of forced scripts against the float64 oracle decode of each distinct (window, script) pair, the finite mask
    exact; the route each B took; CUDA-graph replay against eager stepping at B = 129 and 260."""
    _gpu()
    import copy
    import torch.nn.functional as F
    from oracle import stable_path as SP
    from oracle.whisper_ref import model as WM
    from oracle.whisper_ref.model import ModelDimensions
    from stable_ts_b200.decode import DecodingOptions, decode_windows, enc_select
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    dims = ModelDimensions(n_mels=128, n_audio_ctx=1500, n_audio_state=1280, n_audio_head=20, n_audio_layer=1, n_vocab=51866,
                           n_text_ctx=448, n_text_state=1280, n_text_head=20, n_text_layer=2)
    W, model, gm, tk = _mk(dims, 17)
    m64 = copy.deepcopy(model).double()
    audios = torch.stack([SP.synth_audio(480000, seed=120 + i) for i in range(5)])
    audios[4, 150000:] = 0                                    # a window whose tail is silence
    enc5 = gm.encode(gm.log_mel(audios.cuda()))
    feats = enc5["f32"].view(5, dims.n_audio_ctx, -1).cpu().double()
    steps = 6
    scripts = [SP.synth_token_script(steps, tk.eot, seed=11 + s) for s in range(3)]
    opt = DecodingOptions(language="en", sample_len=steps)
    mel = torch.zeros(dims.n_mels, 3000)                      # (not read: the oracle is given the audio features)
    refs = {}
    with pytest.MonkeyPatch.context() as mp:
        # the oracle's LayerNorm computes in fp32 (a guard for fp16 models); in the float64 model it keeps float64
        mp.setattr(WM.LayerNorm, "forward", lambda self, x: F.layer_norm(x, self.normalized_shape, self.weight, self.bias, self.eps))
        for w in range(5):
            for s in range(3):
                _, _, ex = SP.decode_window(m64, mel, audio_features=feats[w:w + 1], forced_tokens=scripts[s],
                                            return_step_logits=True, sample_len=steps, language="en")
                refs[w, s] = [r.double() for r in ex["step_logits"]]
    want_route = {16: "GEMV", 17: "cluster", 128: "cluster", 129: "GEMM", 260: "GEMM"}
    for B, route in want_route.items():
        enc = enc_select(enc5, [b % 5 for b in range(B)])
        forced = torch.tensor([scripts[b % 3] for b in range(B)], dtype=torch.int32).T.contiguous()
        _, x = decode_windows(gm, tk, enc, opt, forced_tokens=forced, return_step_logits=True, reuse_buffers=True)
        assert len(x["step_logits"]) == steps
        worst = 0.0
        for i, g_all in enumerate(x["step_logits"]):
            g_all = g_all.double().cpu()
            for b in range(B):
                r, g = refs[b % 5, b % 3][i], g_all[b]
                fin = r > -1e30
                assert torch.equal(fin, g > -1e30), (B, b, i)
                worst = max(worst, ((g[fin] - r[fin]).abs().max() / r[fin].abs().max()).item())
        del x
        got_route = _step_route(gm, tk, enc, DecodingOptions(language="en", sample_len=2), decode_windows(
            gm, tk, enc, DecodingOptions(language="en", sample_len=1), reuse_buffers=True)[1]["ckv"])
        print(f"B={B}: step linears on the {'/'.join(sorted(got_route))} route, worst step-logit rel err vs float64 {worst:.2e}")
        assert route in got_route and not got_route & ({"GEMV", "cluster"} - {route}), (B, got_route)
        # the bound of test_gpu_decode.py::test_cross_attention_step_logits_match_float64 (B = 3 and 42)
        assert worst < 2e-5
        if B > 128:
            r_eager, _ = decode_windows(gm, tk, enc, opt, use_graph=False, reuse_buffers=True)
            r_graph, _ = decode_windows(gm, tk, enc, opt, reuse_buffers=True)      # CUDA-graph replay of the same step
            assert [r.tokens for r in r_eager] == [r.tokens for r in r_graph]
            for b in range(B):
                assert r_graph[b].tokens == r_graph[b % 5].tokens
    _report("route boundaries", t0)


def _tiny_windows(W, om, gm, n=5, seed=140):
    from oracle import stable_path as SP
    lens = [480000, 300000, 160000, 480000, 90000]
    audios = [SP.synth_audio(lens[i], seed=seed + i) for i in range(n)]
    pad = torch.zeros(n, 480000)
    for i, a in enumerate(audios):
        pad[i, : len(a)] = a
    mels = [W.pad_or_trim(W.log_mel_spectrogram(a, om.dims.n_mels, padding=480000 - len(a)), 3000) for a in audios]
    return gm.encode(gm.log_mel(pad.cuda())), mels


def test_free_running_greedy_above_128_sequences_matches_the_oracle():
    """tiny.en, B = 130 and 257 tiled from 5 distinct windows: every row's tokens equal the CPU oracle's for its window; then
    B = 257 with ragged prompts and one silent-timestamp mask per row."""
    _gpu()
    from oracle import stable_path as SP
    from stable_ts_b200.decode import DecodingOptions, decode_windows, enc_select
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    W, om, gm, tk = _mk("tiny.en", 4)
    enc5, mels = _tiny_windows(W, om, gm)
    opt = DecodingOptions(language="en", sample_len=32)
    refs = [SP.decode_window(om, m, language="en", sample_len=32)[0] for m in mels]
    for B in (130, 257):
        res, _ = decode_windows(gm, tk, enc_select(enc5, [b % 5 for b in range(B)]), opt, reuse_buffers=True)
        for b in range(B):
            assert res[b].tokens == refs[b % 5].tokens, (B, b)
            assert abs(res[b].avg_logprob - refs[b % 5].avg_logprob) < 1e-3
        print(f"B={B}: free-running greedy tokens equal the oracle's for all rows ({[len(r.tokens) for r in refs]} tokens)")
    g = torch.Generator().manual_seed(9)
    prompts5 = [[], torch.randint(300, 40000, (5,), generator=g).tolist(), torch.randint(300, 40000, (37,), generator=g).tolist(),
                [], torch.randint(300, 40000, (12,), generator=g).tolist()]
    masks5 = torch.zeros(5, 1501, dtype=torch.bool)
    for w in range(5):
        masks5[w, 100 * w + 50: 100 * w + 600] = True
    masks5[3] = False
    refs = [SP.decode_window(om, m, language="en", sample_len=32, prompt=prompts5[w] or None, ts_token_mask=masks5[w])[0]
            for w, m in enumerate(mels)]
    B = 257
    res, _ = decode_windows(gm, tk, enc_select(enc5, [b % 5 for b in range(B)]), opt,
                            prompts=[prompts5[b % 5] for b in range(B)], ts_token_mask=masks5[[b % 5 for b in range(B)]], reuse_buffers=True)
    for b in range(B):
        assert res[b].tokens == refs[b % 5].tokens, ("ragged", b)
        assert abs(res[b].avg_logprob - refs[b % 5].avg_logprob) < 1e-3
    print(f"B={B} with ragged prompts and per-row silent-timestamp masks: tokens equal the oracle's")
    _report("free-running greedy", t0)


def test_temperature_best_of_above_128_sequences_is_the_restated_draw():
    """tiny.en, 30 windows x best_of 5 = 150 sequences at temperature 0.7 with explicit uniforms: every sequence's token at
    every step is the inverse-CDF draw of its uniform over the step logits it returned (row b, uniform[step, b]), EOT
    latched, and its sum_logprob the float64 sum of the log-probs of its picks."""
    _gpu()
    from test_sampler_reference_cpu import restate
    from stable_ts_b200.decode import DecodingOptions, decode_windows, enc_select
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    W, om, gm, tk = _mk("tiny.en", 4)
    enc5, _ = _tiny_windows(W, om, gm)
    n_win, best_of, steps, T = 30, 5, 16, 0.7
    B = n_win * best_of
    u = torch.rand(steps, B, generator=torch.Generator().manual_seed(13))
    res, x = decode_windows(gm, tk, enc_select(enc5, [w % 5 for w in range(n_win)]),
                            DecodingOptions(language="en", sample_len=steps, temperature=T, best_of=best_of),
                            uniform=u, return_step_logits=True)
    tok, sum_lp = x["step_tokens"], x["sum_logprob"]
    logits = [l.cpu().numpy() for l in x["step_logits"]]
    ids = dict(eot=int(tk.eot), ts_begin=int(tk.timestamp_begin), no_timestamps=int(tk.no_timestamps))
    n_drawn = 0
    for b in range(B):
        hist, lp = [], 0.0
        for i in range(x["steps"]):
            # the returned logits are already filtered: only the draw, the EOT latch and the log-prob remain
            ref = restate(logits[i][b], hist, apply_ts_rules=False, temperature=T, u=float(u[i, b]), **ids)
            assert tok[i, b] == ref["token"], (b, i, tok[i, b], ref["token"])
            n_drawn += ref["drawn"] != ref["argmax"] and not ref["was_done"]
            if not ref["was_done"]:
                lp += ref["logprob"]
            hist.append(ref["token"])
        assert abs(sum_lp[b] - lp) <= 2e-5 * (1 + abs(lp)), (b, sum_lp[b], lp)
    assert n_drawn > 0
    print(f"B={B} at T={T}: every token is the restated draw ({n_drawn} draws differ from the argmax); chosen {x['chosen'][:6]}...")
    _report("temperature best_of", t0)
