"""Batched transcription driver for the H100 path (mirror of the per-window body of ``transcribe_stable``,
stable_whisper/whisper_word_level/original_whisper.py:492-710).

The reference walks ONE audio sequentially (its seek depends on the decoded timestamps).  Here independent 30 s windows
(different audios, or static shards of one audio with fixed clip boundaries and no prompt carry-over -- the sharded
setting of SURVEY.md section 8e) are processed B at a time:

    log-mel -> encoder -> KV-cached greedy decode -> segment slicing at timestamp tokens -> batched word timestamps

Mirrored per-window behaviour: non-VAD silence masks -> ``ts_token_mask`` per window (``suppress_ts_tokens``,
original_whisper.py:504-511), silent-window skip (:508-510), the no-speech / log-prob window skip (:537-547), segment
pruning (:604-627), ``max_instant_words`` (:655-663) and the data-dependent seek (:703-710; ``transcribe`` walks every
shard until its end, so speech after the last closed segment of a window is re-decoded exactly as the reference does).
Temperature fallback (``decode_with_fallback``, :349-393) runs batched: only the windows that fail the compression-ratio /
log-prob test are decoded again at the next temperature.  Prompt conditioning (``condition_on_previous_text`` /
``initial_prompt``, :320-323,533,696-698) is carried per shard; windows with prompts of different lengths share a batch
(right-aligned initial tokens, stb_decode_step_ragged).
``nonspeech_skip`` / ``avg_prob_threshold`` (:512-526, :665-675) and ``clip_timestamps`` (the reference's load_sections) are
mirrored too; ``only_voice_freq`` is applied by ``api.transcribe`` to the whole waveform before it gets here
(audio_io.voice_freq_filter).  Out of scope here (reference control plane, SURVEY.md section 2): VAD models, denoisers,
regrouping, and the word-level ``suppress_silence`` re-timing of result.py -- for which ``transcribe(segment_hook=...)`` takes
the reference's own class.
"""
from dataclasses import replace
from typing import List, Optional, Sequence

import numpy as np
import torch

from ._lib import device_ctx
from .decode import DecodingOptions, decode_with_fallback
from .model import B200Whisper
from .timing import add_word_timestamps_batch

SAMPLE_RATE = 16000
N_SAMPLES = 480000
N_SAMPLES_PER_TOKEN = 320
TIME_PRECISION = 0.02


def slice_segments(tokens: Sequence[int], tokenizer, time_offset: float, segment_duration: float, result) -> (List[dict], int):
    """Split one window's sampled tokens into segments at consecutive timestamp tokens
    (original_whisper.py:550-602).  -> (segments, end_timestamp_pos)."""
    tb = tokenizer.timestamp_begin
    toks = list(tokens)
    is_ts = [t >= tb for t in toks]
    single_ending = is_ts[-2:] == [False, True]
    consecutive = [i + 1 for i in range(len(toks) - 1) if is_ts[i] and is_ts[i + 1]]
    seek = round(time_offset * SAMPLE_RATE)

    def seg(start, end, ts):
        text_tokens = [t for t in ts if t < tokenizer.eot]
        return dict(seek=round(seek / SAMPLE_RATE, 3), start=start, end=end, tokens=list(ts), text=tokenizer.decode(text_tokens),
                    temperature=result.temperature, avg_logprob=result.avg_logprob,
                    compression_ratio=result.compression_ratio, no_speech_prob=result.no_speech_prob)

    segments, end_pos = [], 0
    if consecutive:
        slices = consecutive + ([len(toks)] if single_ending else [])
        last = 0
        for cur in slices:
            ts = toks[last:cur]
            s_pos, end_pos = ts[0] - tb, ts[-1] - tb
            segments.append(seg(round(time_offset + s_pos * TIME_PRECISION, 3),
                                round(time_offset + min(end_pos * TIME_PRECISION, segment_duration), 3), ts))
            last = cur
    else:
        duration = segment_duration
        stamps = [t for t in toks if t >= tb]
        if stamps and stamps[-1] != tb:
            end_pos = stamps[-1] - tb
            duration = min(end_pos * TIME_PRECISION, segment_duration)
        segments.append(seg(round(time_offset, 3), round(time_offset + duration, 3), toks))
    return segments, end_pos, single_ending


@torch.no_grad()
def transcribe_windows(model: B200Whisper, tokenizer, audios: Sequence[torch.Tensor], *, time_offsets: Optional[Sequence[float]] = None,
                       word_timestamps: bool = True, options: Optional[DecodingOptions] = None,
                       ts_token_mask: Optional[torch.Tensor] = None, forced_tokens: Optional[torch.Tensor] = None,
                       gap_padding: Optional[str] = " ...", min_word_dur: float = 0.1, punctuations: str = "\"'“¿([{-\"'.。,，!！?？:：”)]}、",
                       enc: Optional[dict] = None, n_samples: Optional[Sequence[int]] = None, use_graph: bool = True,
                       suppress_ts_tokens: bool = False, skip_silent: bool = False, q_levels: int = 20, k_size: int = 5,
                       no_speech_threshold: Optional[float] = None, logprob_threshold: Optional[float] = None,
                       max_instant_words: Optional[float] = None, temperature=0.0,
                       compression_ratio_threshold: Optional[float] = None, prompts=None,
                       generator: Optional[torch.Generator] = None, uniforms=None, nonspeech_skip: Optional[float] = None,
                       avg_prob_threshold: Optional[float] = None, dynamic_heads=None, aligner="legacy", extra_models=None,
                       prepend_punctuations: Optional[str] = None, append_punctuations: Optional[str] = None,
                       split_callback=None):
    """B independent <=30 s windows -> (list (per window) of segment dicts with ``words``, info).
    ``enc`` (+ ``n_samples``) may be passed instead of ``audios`` when the encoder output is already on the device.

    suppress_ts_tokens / skip_silent: run the batched non-VAD silence detector on the windows (silence.py); the former
    feeds one ``ts_token_mask`` row per window to the sampler, the latter drops windows that are entirely silent.
    no_speech_threshold / logprob_threshold / max_instant_words: the reference's per-window filters (transcribe_stable
    defaults 0.6 / -1.0 / 0.5); None here = off, so that fixed-script benchmark windows are never dropped.
    temperature (a number or the fallback sequence) / compression_ratio_threshold / logprob_threshold / no_speech_threshold:
    ``decode_with_fallback`` (original_whisper.py:349-393); prompts: per-window previous-context tokens (:533);
    generator / uniforms: the random stream of the temperature > 0 passes (decode.decode_windows).
    nonspeech_skip: a silence of at least this many seconds ends the window where it starts -- or, when it starts within
    ``min_word_dur`` of the window start, the window is skipped up to the silence's end (original_whisper.py:512-526).
    avg_prob_threshold: a window that ends on a single timestamp and whose words average below it is dropped; otherwise the
    seek moves to the end of the last word (original_whisper.py:665-675,693-694).
    dynamic_heads / aligner / extra_models / prepend_punctuations / append_punctuations / split_callback: the word-timestamp
    options of ``add_word_timestamps_stable`` (original_whisper.py:635-651), passed to the batched alignment pass.
    info["advance"][b]: samples the reference's seek would move by after this window (original_whisper.py:703-710)."""
    dev_audio = None
    if enc is None:
        if torch.is_tensor(audios) and audios.ndim == 2 and audios.shape[1] == N_SAMPLES and audios.dtype == torch.float32:
            batch = audios                                   # already a [B, 480000] batch (ideally pinned): no host copy
            if n_samples is None:
                n_samples = [N_SAMPLES] * batch.shape[0]
        else:
            B = len(audios)
            batch = torch.zeros(B, N_SAMPLES, dtype=torch.float32)
            n_samples = []
            for i, a in enumerate(audios):
                a = a.detach().float().flatten()[:N_SAMPLES]
                batch[i, : a.numel()] = a
                n_samples.append(int(a.numel()))
        if batch.device.type == "cpu" and torch.device(model.device).type == "cuda" and not batch.is_pinned():
            batch = batch.pin_memory()
        with device_ctx(model.device):
            dev_audio = batch.to(model.device, non_blocking=True)
    B = enc["B"] if enc is not None else int(dev_audio.shape[0])
    n_samples = list(n_samples) if n_samples is not None else [N_SAMPLES] * B
    offs = list(time_offsets) if time_offsets is not None else [0.0] * B
    if options is None:                      # transcribe_stable defaults max_initial_timestamp to None (original_whisper.py:262-263)
        options = DecodingOptions(max_initial_timestamp=None)
    silent = [False] * B
    silence_timings = [None] * B                             # (starts, ends) in seconds of every window's silences, or None
    jump = [None] * B                                        # nonspeech_skip: samples to fast-forward instead of decoding
    if suppress_ts_tokens or skip_silent or nonspeech_skip:
        if dev_audio is None:
            raise ValueError("silence detection needs the window audio (pass `audios`, not only `enc`)")
        from .silence import predict_nonvad_batch
        masks = [None] * B
        by_len = {}
        for b, n in enumerate(n_samples):
            by_len.setdefault(n, []).append(b)
        for n, idx in by_len.items():        # the kernel takes equal-length rows: one launch per distinct window length
            rows = dev_audio[idx][:, :n] if len(idx) != B else dev_audio[:, :n]
            for b, pred in zip(idx, predict_nonvad_batch(rows, offsets=[offs[b] for b in idx], q_levels=q_levels, k_size=k_size,
                                                         min_word_dur=min_word_dur)):
                masks[b] = pred["mask"]
                silence_timings[b] = pred["timings"]
                silent[b] = bool(pred["is_silent"]) and skip_silent
                if nonspeech_skip and pred["timings"] is not None and not silent[b]:       # original_whisper.py:512-526
                    starts, ends = pred["timings"][0] - offs[b], pred["timings"][1] - offs[b]
                    long_ones = np.flatnonzero((ends - starts) >= nonspeech_skip)
                    if len(long_ones):
                        k = long_ones[0]
                        if starts[k] < (min_word_dur or 0) or int(starts[k] * SAMPLE_RATE) == 0:
                            jump[b] = round(float(ends[k]) * SAMPLE_RATE)
                        else:                                 # the window ends where the long silence begins
                            n_samples[b] = int(starts[k] * SAMPLE_RATE)
                            if dev_audio is batch:            # the caller's own device tensor: do not write into it
                                dev_audio = dev_audio.clone()
                            dev_audio[b, n_samples[b]:] = 0
        if suppress_ts_tokens and ts_token_mask is None and any(m is not None for m in masks):
            ts_token_mask = masks
    if enc is None:
        with device_ctx(model.device):
            enc = model.encode(model.log_mel(dev_audio))
    # the cross K/V block and the KV cache live in model-owned buffers: they are consumed inside this call (decode loop, then
    # the alignment pass below) and are by far the largest allocations of a step
    results, extras, n_fallback = decode_with_fallback(
        model, tokenizer, enc, options, temperature=temperature, compression_ratio_threshold=compression_ratio_threshold,
        logprob_threshold=logprob_threshold, no_speech_threshold=no_speech_threshold, ts_token_mask=ts_token_mask,
        prompts=prompts, generator=generator, uniforms=uniforms, forced_tokens=forced_tokens, use_graph=use_graph,
        reuse_buffers=True)
    # a re-decode of a subset (or a best_of batch) overwrote the model-owned cross K/V block: the alignment pass rebuilds it
    ckv_valid = not any(n_fallback) and extras.get("n_group", 1) == 1
    windows, advance, skipped, single = [], [], [], []
    for b in range(B):
        dur = n_samples[b] / SAMPLE_RATE
        toks = results[b].tokens if forced_tokens is None else extras["step_tokens"][:, b].tolist()
        skip = silent[b] or jump[b] is not None
        if not skip and no_speech_threshold is not None:          # original_whisper.py:537-547
            skip = results[b].no_speech_prob > no_speech_threshold
            if logprob_threshold is not None and results[b].avg_logprob > logprob_threshold:
                skip = False
        segs, end_pos, single_ending = ([], 0, False)
        if not skip and len(toks):
            segs, end_pos, single_ending = slice_segments(toks, tokenizer, offs[b], dur, results[b])
        # prune punctuation-only and zero-length segments (original_whisper.py:604-627, word_timestamps branch)
        # (`in` on a str is a substring test, so empty-text segments are dropped too, exactly as the reference does)
        segs = [s for s in segs if s["text"].strip() not in punctuations]
        segs = [s for s in segs if not (word_timestamps and s["start"] == s["end"])]
        for s in segs:
            s["seek"] = offs[b]
        num = min(round(end_pos * N_SAMPLES_PER_TOKEN), n_samples[b]) if end_pos > 0 else n_samples[b]
        win = dict(segments=segs, num_samples=num)
        if extra_models and dev_audio is not None:           # every extra model runs its own front end on the window
            win["audio"] = dev_audio[b, : n_samples[b]].cpu()
        windows.append(win)
        advance.append(n_samples[b] if (skip or single_ending or not len(toks)) else num)
        skipped.append(bool(skip))
        single.append(bool(single_ending))
    if word_timestamps:
        add_word_timestamps_batch(windows, model, tokenizer, enc=enc, ckv=extras["ckv"] if ckv_valid else None,
                                  gap_padding=gap_padding, min_word_dur=min_word_dur, dynamic_heads=dynamic_heads,
                                  aligner=aligner, extra_models=extra_models, prepend_punctuations=prepend_punctuations,
                                  append_punctuations=append_punctuations, split_callback=split_callback)
        if max_instant_words is not None:                          # original_whisper.py:655-663
            for w in windows:
                w["segments"] = [s for s in w["segments"] if not s["words"] or float(np.mean(np.array(
                    [x["start"] == x["end"] for x in s["words"]]).astype(np.float16))) <= max_instant_words]
        if avg_prob_threshold:                                     # original_whisper.py:665-675,693-694
            for b, w in enumerate(windows):
                if not w["segments"]:
                    continue
                if single[b] and float(np.mean([x["probability"] for s in w["segments"] for x in s["words"]])) < avg_prob_threshold:
                    w["segments"] = []
                else:
                    advance[b] = round((w["segments"][-1]["words"][-1]["end"] - offs[b]) * SAMPLE_RATE)
    for b, w in enumerate(windows):
        if not w["segments"]:
            advance[b] = n_samples[b]                              # nothing kept: the reference fast-forwards the whole window
        if jump[b] is not None:
            advance[b] = jump[b]                                   # skipped up to the end of a long leading silence
    return [w["segments"] for w in windows], dict(decode=results, steps=extras["steps"], step_argmax=extras["step_argmax"],
                                                  step_tokens=extras["step_tokens"], advance=advance, skipped=skipped,
                                                  silence_timings=silence_timings)


def clip_sections(clip_timestamps, total: int) -> List[List[int]]:
    """``clip_timestamps`` ("s0,e0,s1,e1,..." or a flat list of seconds; an odd count leaves the last clip open) ->
    [[start, end], ...] in samples (original_whisper.py:280-287; audio/__init__.py:431-439: ``round(t * sr)``)."""
    if isinstance(clip_timestamps, str):
        clip_timestamps = [float(t) for t in (clip_timestamps.split(",") if clip_timestamps else [])]
    ts = list(clip_timestamps or [])
    pairs = [ts[i:i + 2] for i in range(0, len(ts), 2)]
    out = []
    for p in pairs:
        lo = round(p[0] * SAMPLE_RATE) if p[0] is not None else 0
        hi = round(p[1] * SAMPLE_RATE) if len(p) == 2 and p[1] is not None else total
        out.append([max(lo, 0), min(hi, total)])
    return out


def transcribe(model: B200Whisper, tokenizer, audio: torch.Tensor, *, initial_prompt: Optional[str] = None, **kw) -> dict:
    """One audio: the one-recording case of ``transcribe_recordings`` (see there for every option).
    -> dict(text, segments, language) in the shape of WhisperResult.to_dict (result.py:1398-1406)."""
    return transcribe_recordings(model, [tokenizer], [audio], initial_prompts=[initial_prompt], **kw)[0]


def transcribe_recordings(model: B200Whisper, tokenizers: Sequence, audios: Sequence[torch.Tensor], *,
                          initial_prompts: Optional[Sequence[Optional[str]]] = None, batch_windows: int = 16,
                          shard_seconds: Optional[float] = 30.0, no_speech_threshold: Optional[float] = 0.6,
                          logprob_threshold: Optional[float] = -1.0, max_instant_words: Optional[float] = 0.5,
                          skip_silent: bool = True, condition_on_previous_text: bool = False, clip_timestamps=None,
                          segment_hook=None, progress_callback=None, options: Optional[DecodingOptions] = None,
                          **kw) -> List[dict]:
    """Several audios, each with its own tokenizer and initial prompt, as static shards in one queue.

    Every audio is cut into static shards (clip boundaries at multiples of ``shard_seconds``, no prompt carry-over: the
    sharded setting of SURVEY.md section 8e).  Inside a shard the walk is the reference's: a window starts at the shard's
    seek, and the seek then moves by the data-dependent amount of original_whisper.py:703-710, so the tail after the last
    closed segment of a window is decoded again by the next window.  Every round takes the tokenizer of the first unfinished
    shard in the queue and batches the current window of up to ``batch_windows`` unfinished shards that share that tokenizer
    (the caller builds one tokenizer per language, so audios in different languages never share a decode batch); shards that
    are not finished go back to the front of the queue.  ``shard_seconds=None``: every audio is one shard (sequential, as the
    reference).  A shard's windows depend only on that shard, so every audio's result equals the one it gets alone, except
    that temperature > 0 draws come from the shared ``generator`` / ``uniforms`` stream in batch order.
    condition_on_previous_text / initial_prompts: the tokens of a shard's kept segments are the prompt of its next window
    (``all_tokens[prompt_reset_since:]``, original_whisper.py:320-323,533,673-675,696-698), reset after a window decoded at
    temperature > 0.5; every shard starts from its audio's initial prompt.
    clip_timestamps: only these [start, end) sections of every audio are transcribed (the reference's ``load_sections``,
    audio/__init__.py:414-429: a window never crosses a section end, and a section is left once ``seek + 1 >= end``).  With
    ``shard_seconds=None`` they are walked in order as ONE shard (shared prompt state, exactly the reference); otherwise every
    clip is a shard of its own and the clips run batched side by side.
    segment_hook(segment_dict, (silent_starts, silent_ends)) -> segment_dict: applied to every kept segment of a window whose
    silences were detected -- where ``api.transcribe`` plugs the reference's own ``Segment.suppress_silence`` re-timing
    (original_whisper.py:677-689) when stable-ts is installed.
    progress_callback(seconds_done, total_seconds): called after every round of windows (the reference's callback,
    original_whisper.py:480-481; with several shards in flight ``seconds_done`` is the audio covered over all shards of all
    audios).
    -> one dict(text, segments, language) per audio, in the shape of WhisperResult.to_dict (result.py:1398-1406); segment
    ``id``s count per audio."""
    audios = [a.detach().float().flatten() for a in audios]
    initial_prompts = list(initial_prompts) if initial_prompts is not None else [None] * len(audios)
    # a shard = the audio it belongs to + a list of [start, end) sections walked in order + the index of the current one +
    # the seek inside it
    rec, plans = [], []
    slack = 1 if clip_timestamps else 0                                  # `seek + 1 >= max_seek` ends a section
    for r, audio in enumerate(audios):
        total = int(audio.numel())
        if clip_timestamps:
            secs = clip_sections(clip_timestamps, total)
            own = [secs] if not shard_seconds else [[sc] for sc in secs]
        else:
            step = total if not shard_seconds else max(int(round(shard_seconds * SAMPLE_RATE)), 1)
            own = [[[lo, min(lo + step, total)]] for lo in range(0, max(total, 1), step)]
        rec += [r] * len(own)
        plans += own
    cur = [0] * len(plans)                                               # current section of every shard
    seek = [p[0][0] if p else 0 for p in plans]

    def settle(i) -> bool:
        """Move shard i to its next section while the current one is exhausted; False when the shard is finished."""
        while cur[i] < len(plans[i]):
            lo, hi = plans[i][cur[i]]
            seek[i] = max(seek[i], lo)
            if seek[i] + slack < hi:
                return True
            cur[i] += 1
        return False

    per_shard = [[] for _ in plans]
    covered = [0] * len(plans)                                           # samples walked per shard (progress reporting)
    span = max(sum(hi - lo for p in plans for lo, hi in p), 1)
    inits = [tokenizers[r].encode(" " + p.strip()) if p is not None else [] for r, p in enumerate(initial_prompts)]
    all_tokens = [list(inits[r]) for r in rec]
    reset_since = [0] * len(plans)
    use_prompts = condition_on_previous_text or any(inits)
    live = [i for i in range(len(plans)) if plans[i] and settle(i)]
    while live:
        tk = tokenizers[rec[live[0]]]
        now = [i for i in live if tokenizers[rec[i]] is tk][:batch_windows]
        taken = set(now)
        live = [i for i in live if i not in taken]
        part = [audios[rec[i]][seek[i]: min(seek[i] + N_SAMPLES, plans[i][cur[i]][1])] for i in now]
        opts = options if options is None else replace(options, language=getattr(tk, "language", None) or options.language)
        segs, info = transcribe_windows(model, tk, part, time_offsets=[seek[i] / SAMPLE_RATE for i in now], options=opts,
                                        no_speech_threshold=no_speech_threshold, logprob_threshold=logprob_threshold,
                                        max_instant_words=max_instant_words, skip_silent=skip_silent,
                                        prompts=[all_tokens[i][reset_since[i]:] for i in now] if use_prompts else None, **kw)
        again = []
        for k, i in enumerate(now):
            if segs[k]:                                       # original_whisper.py:673-675,696-698
                all_tokens[i].extend(t for s in segs[k] for t in s["tokens"])
                if not condition_on_previous_text or info["decode"][k].temperature > 0.5:
                    reset_since[i] = len(all_tokens[i])
                timings = info["silence_timings"][k]
                if segment_hook is not None and timings is not None:               # original_whisper.py:677-689
                    segs[k][:] = [segment_hook(sg, timings) for sg in segs[k]]
            per_shard[i].extend(segs[k])
            covered[i] += max(int(info["advance"][k]), 1)
            seek[i] += max(int(info["advance"][k]), 1)
            if settle(i):
                again.append(i)
        live = again + live
        if progress_callback is not None:
            progress_callback(round(min(sum(covered), span) / SAMPLE_RATE, 2), round(span / SAMPLE_RATE, 2))
    out = []
    for r, tokenizer in enumerate(tokenizers):
        segments = [s for i, ps in enumerate(per_shard) if rec[i] == r for s in ps]
        for k, s in enumerate(segments):
            s["id"] = k
        out.append(dict(text="".join(s["text"] for s in segments), segments=segments,
                        language=getattr(tokenizer, "language", None) or "en"))
    return out
