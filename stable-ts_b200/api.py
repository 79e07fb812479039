"""``load_model`` and the bound model methods (mirror of stable_whisper/whisper_word_level/original_whisper.py:931-1009).

``load_model`` returns a ``B200Whisper`` on which ``modify_model`` has bound ``transcribe`` / ``align`` / ``align_words`` /
``refine`` / ``locate`` -- the names the reference binds at original_whisper.py:942-949 -- and ``transcribe_batch`` (many
recordings through shared device batches, one result each), each returning a WhisperResult
(``result.make_result``: the reference's own class when ``stable_whisper`` is importable, else the schema-compatible
stand-in of ``result.py``).

Control plane: the reference's model-agnostic ``Aligner`` / ``Refiner`` (stable_whisper/non_whisper/alignment.py:58,
refinement.py:13) own the data-dependent window/seek/fallback logic of ``align`` / ``align_words`` / ``refine``; they are
NOT re-implemented here.  When ``stable_whisper`` is importable these methods build exactly the objects the reference's
own entry points build (alignment.py:184-218, 340-367, 612-632) with the H100 plugin closures in place of the PyTorch
ones.  Without the reference package, ``align_words`` and ``transcribe`` (whose windows are known up front) run on the
built-in batched drivers, while ``align`` / ``refine`` raise with the reason.  ``transcribe`` and ``locate`` always run on
the built-in drivers (transcribe.py, locate.py).
"""
import os
import warnings
from types import MethodType
from typing import Optional, Tuple, Union

import torch

from ._lib import device_ctx
from .model import B200Whisper, ModelDimensions
from .result import make_result, result_segments

MODEL_DIMS = {
    "tiny.en": (80, 1500, 384, 6, 4, 51864, 448, 384, 6, 4), "tiny": (80, 1500, 384, 6, 4, 51865, 448, 384, 6, 4),
    "base.en": (80, 1500, 512, 8, 6, 51864, 448, 512, 8, 6), "base": (80, 1500, 512, 8, 6, 51865, 448, 512, 8, 6),
    "small.en": (80, 1500, 768, 12, 12, 51864, 448, 768, 12, 12), "small": (80, 1500, 768, 12, 12, 51865, 448, 768, 12, 12),
    "medium.en": (80, 1500, 1024, 16, 24, 51864, 448, 1024, 16, 24),
    "medium": (80, 1500, 1024, 16, 24, 51865, 448, 1024, 16, 24),
    "large-v1": (80, 1500, 1280, 20, 32, 51865, 448, 1280, 20, 32),
    "large-v2": (80, 1500, 1280, 20, 32, 51865, 448, 1280, 20, 32),
    "large-v3": (128, 1500, 1280, 20, 32, 51866, 448, 1280, 20, 32),
    "large": (128, 1500, 1280, 20, 32, 51866, 448, 1280, 20, 32),
    "large-v3-turbo": (128, 1500, 1280, 20, 32, 51866, 448, 1280, 20, 4),
    "turbo": (128, 1500, 1280, 20, 32, 51866, 448, 1280, 20, 4),
}


def random_state_dict(dims: ModelDimensions, seed: int = 0):
    """Seeded random weights at the true Whisper shapes (checkpoints cannot be downloaded offline).  Key names equal
    openai-whisper's.  Generated on the CPU in fp32 so that every device/process sees identical values."""
    import math
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def lin(name, out_f, in_f, bias=True):
        a = 1.0 / math.sqrt(in_f)
        sd[name + ".weight"] = (2 * torch.rand(out_f, in_f, generator=g) - 1) * a
        if bias:
            sd[name + ".bias"] = (2 * torch.rand(out_f, generator=g) - 1) * a

    def ln(name, d):
        sd[name + ".weight"] = 1.0 + 0.1 * (2 * torch.rand(d, generator=g) - 1)
        sd[name + ".bias"] = 0.05 * (2 * torch.rand(d, generator=g) - 1)

    def block(p, d, cross):
        for n in ("attn",) + (("cross_attn",) if cross else ()):
            lin(f"{p}.{n}.query", d, d)
            lin(f"{p}.{n}.key", d, d, bias=False)
            lin(f"{p}.{n}.value", d, d)
            lin(f"{p}.{n}.out", d, d)
            ln(f"{p}.{n}_ln", d)
        lin(f"{p}.mlp.0", 4 * d, d)
        lin(f"{p}.mlp.2", d, 4 * d)
        ln(f"{p}.mlp_ln", d)

    da, dt = dims.n_audio_state, dims.n_text_state
    a1, a2 = 1.0 / math.sqrt(3 * dims.n_mels), 1.0 / math.sqrt(3 * da)
    sd["encoder.conv1.weight"] = (2 * torch.rand(da, dims.n_mels, 3, generator=g) - 1) * a1
    sd["encoder.conv1.bias"] = (2 * torch.rand(da, generator=g) - 1) * a1
    sd["encoder.conv2.weight"] = (2 * torch.rand(da, da, 3, generator=g) - 1) * a2
    sd["encoder.conv2.bias"] = (2 * torch.rand(da, generator=g) - 1) * a2
    half = da // 2
    inv = torch.exp(-(math.log(10000.0) / (half - 1)) * torch.arange(half))
    st = torch.arange(dims.n_audio_ctx)[:, None] * inv[None, :]
    sd["encoder.positional_embedding"] = torch.cat([torch.sin(st), torch.cos(st)], dim=1)
    for l in range(dims.n_audio_layer):
        block(f"encoder.blocks.{l}", da, False)
    ln("encoder.ln_post", da)
    sd["decoder.token_embedding.weight"] = torch.randn(dims.n_vocab, dt, generator=g) * 0.05
    sd["decoder.positional_embedding"] = torch.randn(dims.n_text_ctx, dt, generator=g) * 0.05
    for l in range(dims.n_text_layer):
        block(f"decoder.blocks.{l}", dt, True)
    ln("decoder.ln", dt)
    return sd


# Cross-attention alignment heads of the released checkpoints as (decoder layer, head) pairs: openai-whisper's
# ``_ALIGNMENT_HEADS`` table (whisper/__init__.py, applied by ``whisper.load_model`` via ``model.set_alignment_heads``).
# Recalled from the published per-model tables (the same pairs ship in the Hugging Face ``generation_config.json``
# ``alignment_heads`` of each checkpoint); nothing in this offline image holds a copy to diff against, so re-verify
# against a real openai-whisper install when one is available.
ALIGNMENT_HEADS = {
    "tiny.en": [(1, 0), (2, 0), (2, 5), (3, 0), (3, 1), (3, 2), (3, 3), (3, 4)],
    "tiny": [(2, 2), (3, 0), (3, 2), (3, 3), (3, 4), (3, 5)],
    "base.en": [(3, 3), (4, 7), (5, 1), (5, 5), (5, 7)],
    "base": [(3, 1), (4, 2), (4, 3), (4, 7), (5, 1), (5, 2), (5, 4), (5, 6)],
    "small.en": [(6, 6), (7, 0), (7, 3), (7, 8), (8, 2), (8, 5), (8, 7), (9, 0), (9, 4), (9, 8), (9, 10), (10, 0), (10, 1),
                 (10, 2), (10, 3), (10, 6), (10, 11), (11, 2), (11, 4)],
    "small": [(5, 3), (5, 9), (8, 0), (8, 4), (8, 7), (8, 8), (9, 0), (9, 7), (9, 9), (10, 5)],
    "medium.en": [(11, 4), (14, 1), (14, 12), (14, 14), (15, 4), (16, 0), (16, 4), (16, 9), (17, 12), (17, 14), (18, 7),
                  (18, 10), (18, 15), (20, 0), (20, 3), (20, 9), (20, 14), (21, 12)],
    "medium": [(13, 15), (15, 4), (15, 15), (16, 1), (20, 0), (23, 4)],
    "large-v1": [(9, 19), (11, 2), (11, 4), (11, 17), (22, 7), (22, 11), (22, 17), (23, 2), (23, 15)],
    "large-v2": [(10, 12), (13, 17), (16, 11), (16, 12), (16, 13), (17, 15), (17, 16), (18, 4), (18, 11), (18, 19), (19, 11),
                 (21, 2), (21, 3), (22, 3), (22, 9), (22, 12), (23, 5), (23, 7), (23, 13), (25, 5), (26, 1), (26, 12), (27, 15)],
    "large-v3": [(7, 0), (10, 17), (12, 18), (13, 12), (16, 1), (17, 14), (19, 11), (21, 4), (24, 1), (25, 6)],
    "large": [(7, 0), (10, 17), (12, 18), (13, 12), (16, 1), (17, 14), (19, 11), (21, 4), (24, 1), (25, 6)],
    "large-v3-turbo": [(2, 4), (2, 11), (3, 3), (3, 6), (3, 11), (3, 14)],
    "turbo": [(2, 4), (2, 11), (3, 3), (3, 6), (3, 11), (3, 14)],
}


def load_model(name: str = "base", device: Optional[Union[str, torch.device]] = None, download_root: str = None,
               in_memory: bool = False, cpu_preload: bool = True, dq: bool = False, engine: Optional[str] = None, *,
               precision: str = "fp16x3", seed: int = 0, allow_random: Optional[bool] = None) -> B200Whisper:
    """Same signature as the reference's ``load_model`` (original_whisper.py:953-955) + ``precision`` / ``seed`` /
    ``allow_random``.

    ``name``: an official model name or a path to an openai-whisper ``.pt`` checkpoint
    (``{"dims": ..., "model_state_dict": ...}``).  For a model NAME the checkpoint is looked up in ``download_root``
    (default ``~/.cache/whisper``).  There is no network here: when the file is absent the model is built with seeded
    random weights at the named shapes, ``model.random_init`` is set and a warning is raised -- pass
    ``allow_random=True`` to silence it (benchmarks, tests) or ``allow_random=False`` to make it an error.
    Named models get the released alignment-head table; other checkpoints set ``missing_alignment_heads`` so that the
    aligner falls back to dynamic head selection (stable_whisper/timing.py:85), as the reference does."""
    if dq:
        raise ValueError("dq (CPU dynamic quantisation) does not apply to the H100 path")
    if engine not in (None, "b200"):
        raise ValueError(f"engine={engine!r}: this package only provides the H100 engine")
    device = device or "cuda"
    is_path = os.path.isfile(name)
    path = name if is_path else os.path.join(download_root or os.path.expanduser("~/.cache/whisper"), f"{name}.pt")
    key = os.path.splitext(os.path.basename(name))[0] if is_path else name
    heads = ALIGNMENT_HEADS.get(key)
    if os.path.isfile(path):
        ckpt = torch.load(path, map_location="cpu", weights_only=True)
        dims = ModelDimensions(**ckpt["dims"])
        if heads is not None and any(l >= dims.n_text_layer or h >= dims.n_text_head for l, h in heads):
            heads = None
        model = B200Whisper(dims, ckpt["model_state_dict"], device=device, precision=precision, alignment_heads=heads)
        model.random_init = False
    else:
        if name not in MODEL_DIMS:
            raise RuntimeError(f"Model {name} not found; available models = {list(MODEL_DIMS)}")
        if allow_random is False:
            raise FileNotFoundError(f"checkpoint {path} not found (and allow_random=False)")
        if allow_random is None:
            warnings.warn(f"checkpoint {path} not found: building '{name}' with SEEDED RANDOM weights (seed={seed}); outputs are "
                          "only meaningful for benchmarks and parity tests.  Pass allow_random=True to silence this.")
        dims = ModelDimensions(*MODEL_DIMS[name])
        model = B200Whisper(dims, random_state_dict(dims, seed), device=device, precision=precision, alignment_heads=heads)
        model.random_init = True
    model.missing_alignment_heads = heads is None
    model.name = name
    return modify_model(model)


# ---------------------------------------------------------------------------------------------------------------------
# bound methods (original_whisper.py:931-949)
# ---------------------------------------------------------------------------------------------------------------------
def _reference():
    """The reference package's control-plane classes, or None when it is not installed."""
    try:
        from stable_whisper.non_whisper.alignment import Aligner
        from stable_whisper.non_whisper.refinement import Refiner
        from stable_whisper.options import AllOptions
        from stable_whisper.result import WhisperResult
        return dict(Aligner=Aligner, Refiner=Refiner, AllOptions=AllOptions, WhisperResult=WhisperResult)
    except Exception:
        return None


def _need_reference(what: str):
    ref = _reference()
    if ref is None:
        raise RuntimeError(
            f"{what}() needs the reference's model-agnostic control plane (stable_whisper.non_whisper Aligner/Refiner: "
            "data-dependent windowing, fallback and silence logic that this package deliberately does not re-implement). "
            "Install stable-ts next to this package, or use align_words()/transcribe(), which run on the built-in drivers.")
    return ref


def _tokenizer_for(model, language: Optional[str], tokenizer=None, text=None):
    """get_alignment_tokenizer (alignment.py:369-386) over this package's tokenizer."""
    from .tokenizer import get_tokenizer
    if tokenizer is not None:
        return tokenizer
    if language is None:
        language = getattr(text, "language", None)
    if language is None:
        if model.is_multilingual:
            raise TypeError("expected argument for language")
        language = "en"
    return get_tokenizer(model, language=language, task="transcribe", synthetic=getattr(model, "random_init", False))


def _as_waveform(audio, model=None) -> torch.Tensor:
    """path | bytes | ndarray | Tensor -> fp32 mono 16 kHz CPU tensor (audio_io.load_audio does the decoding and the
    GPU resampling; arrays are taken as 16 kHz already, as the reference documents)."""
    if isinstance(audio, (str, bytes, os.PathLike)):
        from .audio_io import load_audio
        return load_audio(audio, device=None if model is None else model.device).cpu()
    if not torch.is_tensor(audio):
        import numpy as np
        audio = torch.from_numpy(np.ascontiguousarray(audio))
    return audio.detach().float().flatten().cpu()


def _voice_freq(wave: torch.Tensor, model) -> torch.Tensor:
    """``only_voice_freq=True``: the reference's voice-band filter (audio_io.voice_freq_filter) over the whole waveform,
    run on the model's device and returned on the host, where the drivers take the waveform from."""
    from . import audio_io
    with device_ctx(model.device):
        return audio_io.voice_freq_filter(wave.to(model.device)).cpu()


def _set_language(result, tokenizer, language):
    lang = getattr(tokenizer, "language_code", None) or getattr(tokenizer, "language", None) or language
    try:
        result.language = lang
    except Exception:
        pass
    return result


def _detect_languages(model: B200Whisper, waves, batch_windows: int):
    """``model.detect_language_of(wave[:480000])`` of every waveform, with up to ``batch_windows`` first 30 s per log-mel /
    encoder / language-token pass.  A shorter first 30 s is zero-filled up to the longest one of its batch: the log-mel
    zero-pads every row to 30 s anyway, so a row's mel -- and with it the encoder and decoder rows -- is the one it gets alone."""
    found = []
    step = max(int(batch_windows), 1)
    for lo in range(0, len(waves), step):
        heads = [w[:480000] for w in waves[lo:lo + step]]
        rows = torch.zeros(len(heads), max(int(h.numel()) for h in heads))
        for b, h in enumerate(heads):
            rows[b, : h.numel()] = h
        _, probs = model.detect_language(model.log_mel(rows.to(model.device)))
        found += [max(p, key=p.get) for p in probs]
    return found


def transcribe(model: B200Whisper, audio, *, language: Optional[str] = None, initial_prompt: Optional[str] = None, **options):
    """``model.transcribe`` (transcribe_stable, original_whisper.py:27-78): -> WhisperResult.  The one-recording case of
    ``transcribe_batch``; every option and its default is listed at ``_transcribe``."""
    return _transcribe(model, [audio], [language], [initial_prompt], **options)[0]


def transcribe_batch(model: B200Whisper, audios, *, language=None, initial_prompt=None, **options):
    """``model.transcribe_batch``: many recordings -> one WhisperResult per recording, in input order.

    Every recording's windows join one queue of device batches (transcribe.transcribe_recordings), so short recordings share
    decode steps instead of each running at batch 1.  ``audios``: a sequence of anything ``transcribe`` takes (path, bytes,
    ndarray, tensor).  ``language`` / ``initial_prompt``: one value for every recording or a list with one entry per
    recording; ``None`` in a ``language`` list detects that recording's language (on its first 30 s, batched).  Recordings of
    different languages never share a decode batch.  Every other option is shared and means what it means in ``transcribe``;
    ``progress_callback`` counts over all recordings.  ``clip_timestamps`` is refused (one clip list means nothing across
    different recordings), and so is ``tokenizer`` together with a language list.

    ``transcribe_batch(audios, **kw)[i]`` equals ``transcribe(audios[i], **kw_i)``, ``kw_i`` being ``kw`` with that recording's
    language and initial prompt -- segments, seeks, tokens and word times, word probabilities up to the decode-step route
    that the batch size selects -- as long as no window falls back to a temperature above 0: the draws of such windows come
    from the shared ``generator`` / ``uniforms`` stream in batch order."""
    audios = list(audios)

    def per_recording(name, value):
        if not isinstance(value, (list, tuple)):
            return [value] * len(audios)
        if len(value) != len(audios):
            raise ValueError(f"transcribe_batch: {len(value)} entries in {name} for {len(audios)} recordings")
        return list(value)
    if options.get("clip_timestamps") is not None:
        raise TypeError("transcribe_batch does not take clip_timestamps (one clip list means nothing across recordings)")
    if options.get("tokenizer") is not None and isinstance(language, (list, tuple)):
        raise ValueError("transcribe_batch: pass either tokenizer= or a per-recording language list, not both")
    return _transcribe(model, audios, per_recording("language", language), per_recording("initial_prompt", initial_prompt),
                       **options)


def _transcribe(model: B200Whisper, audios, languages, initial_prompts, *, task: str = "transcribe",
                word_timestamps: bool = True, regroup=True, suppress_silence: bool = True, suppress_word_ts: bool = True,
                use_word_position: bool = True, nonspeech_error: float = 0.1, suppress_ts_tokens: bool = False,
                q_levels: int = 20, k_size: int = 5, temperature: Union[float, Tuple[float, ...]] = (0.0, 0.2, 0.4, 0.6, 0.8, 1.0),
                compression_ratio_threshold: Optional[float] = 2.4, no_speech_threshold: Optional[float] = 0.6,
                logprob_threshold: Optional[float] = -1.0, condition_on_previous_text: bool = True,
                max_instant_words: Optional[float] = 0.5, gap_padding: str = " ...", min_word_dur: float = 0.1,
                batch_windows: int = 16, shard_seconds: Optional[float] = 30.0, tokenizer=None,
                nonspeech_skip: Optional[float] = None, avg_prob_threshold: Optional[float] = None, clip_timestamps=None,
                dynamic_heads=None, aligner="legacy", extra_models=None, prepend_punctuations: Optional[str] = None,
                append_punctuations: Optional[str] = None, split_callback=None, progress_callback=None,
                verbose: Optional[bool] = False, ignore_compatibility: bool = False, only_voice_freq: bool = False,
                generator: Optional[torch.Generator] = None, uniforms=None, **decode_options):
    """``transcribe`` / ``transcribe_batch`` over recordings ``audios`` with one language (None: detect) and one initial
    prompt each -> one WhisperResult per recording.  Static 30 s shards batched ``batch_windows`` at a time
    (transcribe.py); ``shard_seconds=None`` walks each recording as one sequential shard like the reference.  Decoding
    defaults are the reference's: the temperature fallback sequence with its compression-ratio / log-prob / no-speech tests,
    ``best_of`` draws at temperature > 0, the previous window's text as the prompt of the next (inside a shard).
    ``suppress_silence``: as in the reference (original_whisper.py:428) the non-VAD silence detector only runs when it is
    True -- silent windows are then skipped and ``suppress_ts_tokens`` masks the silent timestamp tokens.  The word
    re-timing against the detected silences (``Segment.suppress_silence``, result.py; governed by ``suppress_word_ts`` /
    ``use_word_position`` / ``nonspeech_error``) is the reference's own code: it is applied per window exactly where the
    reference applies it (original_whisper.py:677-689) when stable-ts is installed, and skipped -- with a warning -- when it is
    not (result post-processing is outside this package's scope).  ``generator`` / ``uniforms``: random stream of the
    temperature > 0 passes (decode.decode_with_fallback).  Beam search is not implemented.
    ``progress_callback(seconds_done, total_seconds)`` as in the reference; ``verbose=True`` prints the segments;
    ``ignore_compatibility`` is accepted for call compatibility (there is no whisper version to check).
    ``only_voice_freq``: band-limit the waveform to 200-5000 Hz first (audio_io.voice_freq_filter), so that language
    detection, the silence detector, the log-mel and the decode all see the filtered audio, as in the reference.
    A multilingual model detects the language of every recording without one on its first 30 s (``_detect_languages``)."""
    from .decode import DecodingOptions
    from .tokenizer import get_tokenizer
    from .transcribe import transcribe_recordings
    if decode_options.get("beam_size") is not None:
        raise NotImplementedError("H100 transcribe: beam search is not implemented (greedy / temperature sampling only)")
    if decode_options.pop("prompt", None):
        raise TypeError("transcribe: use initial_prompt (the per-window prompt is managed by condition_on_previous_text)")
    waves = [_as_waveform(audio, model) for audio in audios]
    if only_voice_freq:
        waves = [_voice_freq(wave, model) for wave in waves]
    languages = [lang if lang is not None or model.is_multilingual else "en" for lang in languages]
    undetected = [r for r, lang in enumerate(languages) if lang is None]
    for r, lang in zip(undetected, _detect_languages(model, [waves[r] for r in undetected], batch_windows)):
        languages[r] = lang
    tokenizers = {}                                    # one per language: the scheduler batches recordings that share one
    for lang in languages:
        if lang not in tokenizers:
            tokenizers[lang] = tokenizer or get_tokenizer(model, language=lang, task=task,
                                                          synthetic=getattr(model, "random_init", False))
    unknown = sorted(k for k in decode_options if k not in DecodingOptions.__dataclass_fields__)
    if unknown:                                        # the reference hands them to DecodingOptions(**kwargs), which raises too
        raise TypeError(f"transcribe() got unexpected decoding option(s): {unknown}")
    opts = DecodingOptions(task=task, language=languages[0] if languages else None,
                           max_initial_timestamp=decode_options.pop("max_initial_timestamp", None), **decode_options)
    hook = None
    if suppress_silence and word_timestamps:
        try:
            from stable_whisper.result import Segment as _RefSegment

            def hook(seg: dict, timings):
                return _RefSegment(**seg, ignore_unused_args=True).suppress_silence(
                    *timings, min_word_dur=min_word_dur, word_level=suppress_word_ts, nonspeech_error=nonspeech_error,
                    use_word_position=use_word_position).to_dict()
        except Exception:
            warnings.warn("stable-ts is not installed: the words are not re-timed against the detected silences "
                          "(suppress_silence only gates the silence detector here)")
    done = transcribe_recordings(
        model, [tokenizers[lang] for lang in languages], waves, initial_prompts=initial_prompts, batch_windows=batch_windows,
        shard_seconds=shard_seconds, word_timestamps=word_timestamps, options=opts,
        suppress_ts_tokens=bool(suppress_ts_tokens and suppress_silence), skip_silent=bool(suppress_silence),
        q_levels=q_levels, k_size=k_size, no_speech_threshold=no_speech_threshold, logprob_threshold=logprob_threshold,
        max_instant_words=max_instant_words, gap_padding=gap_padding, min_word_dur=min_word_dur, temperature=temperature,
        compression_ratio_threshold=compression_ratio_threshold, condition_on_previous_text=condition_on_previous_text,
        generator=generator, uniforms=uniforms, nonspeech_skip=nonspeech_skip if suppress_silence else None,
        avg_prob_threshold=avg_prob_threshold, clip_timestamps=clip_timestamps, segment_hook=hook,
        dynamic_heads=dynamic_heads, aligner=aligner, extra_models=extra_models, prepend_punctuations=prepend_punctuations,
        append_punctuations=append_punctuations, split_callback=split_callback, progress_callback=progress_callback)
    results = []
    for d, lang in zip(done, languages):
        d["language"] = lang
        if verbose:                                    # the reference prints every segment as it is produced; here at the end
            for sg in d["segments"]:
                print(f"[{sg['start']:.3f} --> {sg['end']:.3f}] {sg['text']}")
        res = make_result(d)
        if regroup and hasattr(res, "regroup") and word_timestamps:
            res.regroup(regroup)
        results.append(res)
    return results


def align(model: B200Whisper, audio, text, language: Optional[str] = None, *, tokenizer=None, remove_instant_words: bool = False,
          token_step: int = 100, original_split: bool = False, word_dur_factor: Optional[float] = 2.0,
          max_word_dur: Optional[float] = 3.0, nonspeech_skip: Optional[float] = 5.0, fast_mode: bool = False,
          failure_threshold: Optional[float] = None, **options):
    """``model.align`` (alignment.py:27-218): the reference's ``Aligner`` over the H100 alignment closure."""
    ref = _need_reference("align")
    from .alignment import N_SAMPLES, get_b200_alignment_func
    max_token_step = model.dims.n_text_ctx - 6
    if token_step < 1:
        token_step = max_token_step
    elif token_step > max_token_step:
        raise ValueError(f"The max value for [token_step] is {max_token_step} but got {token_step}.")
    tk = _tokenizer_for(model, language, tokenizer, text)
    opts = ref["AllOptions"](options, vanilla_align=True)
    by_space = getattr(tk, "language_code", getattr(tk, "language", None)) not in {"zh", "ja", "th", "lo", "my"}
    aligner = ref["Aligner"](inference_func=get_b200_alignment_func(model, tk, opts), decode=tk.decode, encode=tk.encode,
                             split_words_by_space=by_space, sample_rate=16000, tokens_per_sec=50, max_segment_length=N_SAMPLES,
                             remove_instant_words=remove_instant_words, token_step=token_step, original_split=original_split,
                             word_dur_factor=word_dur_factor, max_word_dur=max_word_dur, nonspeech_skip=nonspeech_skip,
                             fast_mode=fast_mode, failure_threshold=failure_threshold, all_options=opts)
    audio = audio if not isinstance(audio, (str, bytes, os.PathLike)) else _as_waveform(audio, model)
    return _set_language(aligner.align(audio, text), tk, language)


def align_words(model: B200Whisper, audio, result, language: Optional[str] = None, *, tokenizer=None, normalize_text: bool = True,
                inplace: bool = True, **options):
    """``model.align_words`` (alignment.py:221-367): every segment is one window confined to its [start, end].  With the
    reference installed its ``Aligner.align_words`` drives the H100 closure segment by segment; without it all segments run
    as ONE batch on the built-in driver (no silence suppression / regrouping afterwards), which takes ``only_voice_freq``
    (audio_io.voice_freq_filter over the whole waveform before the segments are cut) and no other option."""
    from .alignment import N_SAMPLES, align_words_batch, get_b200_alignment_func
    tk = _tokenizer_for(model, language, tokenizer, result)
    ref = _reference()
    if ref is not None:
        opts = ref["AllOptions"](options)
        by_space = getattr(tk, "language_code", getattr(tk, "language", None)) not in {"zh", "ja", "th", "lo", "my"}
        aligner = ref["Aligner"](inference_func=get_b200_alignment_func(model, tk, opts), decode=tk.decode, encode=tk.encode,
                                 split_words_by_space=by_space, sample_rate=16000, max_segment_length=N_SAMPLES,
                                 time_precision=1 / 50, token_step=model.dims.n_text_ctx, all_options=opts)
        audio = audio if not isinstance(audio, (str, bytes, os.PathLike)) else _as_waveform(audio, model)
        return _set_language(aligner.align_words(audio, result, normalize_text, inplace), tk, language)
    only_voice_freq = options.pop("only_voice_freq", False)
    if options:
        raise TypeError(f"align_words without the reference package takes no extra options, got {sorted(options)}")
    wave = _as_waveform(audio, model)
    if only_voice_freq:
        wave = _voice_freq(wave, model)
    segs = [s for s in result_segments(result)]
    audios, groups, names, keep = [], [], [], []
    for i, s in enumerate(segs):
        lo, hi = round(float(s["start"]) * 16000), round(float(s["end"]) * 16000)
        if hi <= lo:
            continue
        toks = [t for t in (s.get("tokens") or tk.encode(s["text"])) if t < tk.eot]
        words, wtoks = tk.split_to_word_tokens(list(toks) + [tk.eot])
        audios.append(wave[lo:min(hi, lo + N_SAMPLES)])
        groups.append([list(w) for w in wtoks[:-1]])
        names.append(list(words[:-1]))
        keep.append(i)
    timed = align_words_batch(model, tk, audios, groups, names) if audios else []
    out = []
    for i, ws in zip(keep, timed):
        off = float(segs[i]["start"])
        words = [dict(w, start=round(off + w["start"], 3), end=round(off + w["end"], 3)) for w in ws]
        out.append(dict(segs[i], words=words, start=words[0]["start"] if words else segs[i]["start"],
                        end=words[-1]["end"] if words else segs[i]["end"]))
    d = dict(segments=out, language=getattr(tk, "language", language))
    return make_result(d)


def refine(model: B200Whisper, audio, result, *, steps: str = None, rel_prob_decrease: float = .03, abs_prob_decrease: float = .05,
           rel_rel_prob_decrease: Optional[float] = None, prob_threshold: float = .5, rel_dur_change: Optional[float] = .5,
           abs_dur_change: Optional[float] = None, word_level: bool = True, precision: float = None, single_batch: bool = False,
           inplace: bool = True, **options):
    """``model.refine`` (alignment.py:512-635): the reference's ``Refiner`` over the H100 refinement closure, which returns the
    3-D probability tensor on the device, so the token-rank test of refinement.py:305-325,427 is live."""
    ref = _need_reference("refine")
    from .alignment import get_b200_refinement_func
    if result and (not result.has_words or any(w.probability is None for w in result.all_words())):
        if not result.language:
            raise RuntimeError("cannot align words with result missing language")
        align_words(model, audio, result)
    tk = _tokenizer_for(model, result.language, None, result)
    if result and not all(w.tokens for w in result.all_words()):
        for w in result.all_words():
            w.tokens = tk.encode(w.word)
    opts = ref["AllOptions"](options, post=False, silence=False, align=False)
    refiner = ref["Refiner"](inference_func=get_b200_refinement_func(model, tk), sample_rate=16000, steps=steps,
                             rel_prob_decrease=rel_prob_decrease, abs_prob_decrease=abs_prob_decrease,
                             rel_rel_prob_decrease=rel_rel_prob_decrease, prob_threshold=prob_threshold,
                             rel_dur_change=rel_dur_change, abs_dur_change=abs_dur_change, word_level=word_level,
                             precision=precision, max_inference_tokens=model.dims.n_text_ctx - 6, all_options=opts)
    audio = audio if not isinstance(audio, (str, bytes, os.PathLike)) else _as_waveform(audio, model)
    return refiner.refine(audio, result, inplace)


def locate(model: B200Whisper, audio, text, language: str, count: int = 1, duration_window=3.0, **kw):
    """``model.locate`` (alignment.py:756-1116), built-in driver (locate.py)."""
    from .locate import locate as run
    return run(model, _as_waveform(audio, model), text, language, count, duration_window, **kw)


def modify_model(model: B200Whisper) -> B200Whisper:
    """Bind the user-facing methods on the model object, as the reference does (original_whisper.py:931-949)."""
    model.transcribe = MethodType(transcribe, model)
    model.transcribe_minimal = MethodType(transcribe, model)
    model.transcribe_batch = MethodType(transcribe_batch, model)
    model.align = MethodType(align, model)
    model.align_words = MethodType(align_words, model)
    model.refine = MethodType(refine, model)
    model.locate = MethodType(locate, model)
    return model
