"""``model.transcribe_batch`` in the build container: many recordings through one queue of device batches must give every
recording exactly what ``model.transcribe`` gives it alone, and what the UNMODIFIED ``transcribe_stable`` gives it, over the
oracle-backed stand-in for the model and the step engine (tests/standin.py).  Also: recordings of different languages never
share a decode batch, and the argument errors of the batch form."""
import os
import sys

import pytest
import torch

REFERENCE = "/root/reference"
pytestmark = pytest.mark.skipif(not os.path.isdir(REFERENCE), reason="reference tree only exists in the build container")

PROMPTS = ["hello there", None, "a longer initial prompt for the third", "more words"]


@pytest.fixture(scope="module")
def env():
    import oracle.whisper_ref as W
    W.install_as_whisper()
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    import stable_whisper  # noqa: F401
    from oracle import stable_path as SP
    from standin import OracleBackedModel, OracleStepEngine
    from stable_ts_b200 import api

    def stand_in(om):
        st = OracleBackedModel(om)
        st.step_engine_cls = OracleStepEngine
        return api.modify_model(st)
    om = W.build_model("tiny.en", seed=3)
    # the silence detector's device stage has no CPU path in the product: stand in with the oracle's restatement (the kernel
    # itself is pinned bit-exactly by tests/test_gpu_silence.py)
    import numpy as np
    import stable_ts_b200.silence as sil
    from oracle import silence as SIL

    def sound_masks(audio, q_levels=20, k_size=5, want_loudness=False):
        audio = audio[None] if audio.ndim == 1 else audio
        if round(audio.shape[1] / 320) + 1 <= 2:
            return None, None
        loud = [SIL.audio2loudness(a.numpy()) for a in audio]
        return np.stack([SIL.loudness_to_raw_mask(l, q_levels, k_size) for l in loud]), (np.stack(loud) if want_loudness else None)
    saved = sil.sound_masks
    sil.sound_masks = sound_masks
    # ~7 s, ~31 s (with gaps), ~65 s (a 4 s silent gap inside) and ~12 s; float32 so that every window is a view of its
    # recording (the spy below maps windows to recordings by storage)
    recs = [SP.synth_audio(112000, seed=101), SP.synth_gapped_audio(496000, seed=102),
            torch.cat([SP.synth_audio(500000, seed=103), torch.zeros(64000), SP.synth_audio(476000, seed=104)]),
            SP.synth_audio(192000, seed=105)]
    recs = [r.float().contiguous() for r in recs]
    yield dict(W=W, om=om, stand=stand_in(om), stand_ml=stand_in(W.build_model("tiny", seed=5)), recs=recs)
    sil.sound_masks = saved


def _assert_same(da, db, rel):
    assert len(da["segments"]) == len(db["segments"])
    for sa, sb in zip(da["segments"], db["segments"]):
        assert sa["tokens"] == [int(t) for t in sb["tokens"]] and sa["seek"] == sb["seek"]
        assert sa["start"] == sb["start"] and sa["end"] == sb["end"]
        assert [w["tokens"] for w in sa["words"]] == [w["tokens"] for w in sb["words"]]
        for wa, wb in zip(sa["words"], sb["words"]):
            assert wa["start"] == wb["start"] and wa["end"] == wb["end"], (wa, wb)
            assert abs(wa["probability"] - wb["probability"]) <= rel * abs(wb["probability"])


# The stand-in's encoder and teacher-forced decoder are fp32 CPU matmuls whose blocking follows the batch size, so the same
# window's word probabilities move by ~1e-6 relative between a batch of 1 and a batch of 3; the bound leaves 7x room.
REL = 1e-5
KW = dict(temperature=0.0, sample_len=16, suppress_silence=True, condition_on_previous_text=True, regroup=False)


@pytest.mark.parametrize("shard_seconds", [30.0, None])
@pytest.mark.parametrize("batch_windows", [1, 3, 16])
def test_batch_equals_separate_calls(env, batch_windows, shard_seconds):
    stand, recs = env["stand"], env["recs"]
    kw = dict(KW, batch_windows=batch_windows, shard_seconds=shard_seconds)
    seen = []
    stand.calls.clear()
    batch = stand.transcribe_batch(recs, language="en", initial_prompt=PROMPTS,
                                   progress_callback=lambda done, total: seen.append((done, total)), **kw)
    n_batched = stand.calls["encode"]
    assert len(batch) == len(recs)
    total = round(sum(r.numel() for r in recs) / 16000, 2)
    assert seen[-1] == (total, total) and all(a[0] <= b[0] for a, b in zip(seen, seen[1:]))
    stand.calls.clear()
    n_segments = 0
    for rec, prompt, got in zip(recs, PROMPTS, batch):
        alone = stand.transcribe(rec, language="en", initial_prompt=prompt, **kw).to_dict()
        da = got.to_dict()
        _assert_same(da, alone, REL)
        assert da["text"] == alone["text"] and da["language"] == "en"
        n_segments += len(da["segments"])
    assert n_segments >= 6
    if batch_windows > 1:                                  # the recordings really shared encoder passes
        assert n_batched < stand.calls["encode"]


def test_batch_equals_unmodified_reference(env):
    """Sequential walk (``shard_seconds=None``): every recording of the batch equals ``transcribe_stable`` on it alone,
    prompt, silence masks and re-timed words included."""
    import stable_whisper.whisper_word_level.original_whisper as ow
    om, stand, recs = env["om"], env["stand"], env["recs"]
    batch = stand.transcribe_batch(recs, language="en", initial_prompt=PROMPTS, batch_windows=16, shard_seconds=None,
                                   suppress_ts_tokens=True, **KW)
    for rec, prompt, got in zip(recs, PROMPTS, batch):
        theirs = ow.transcribe_stable(om, rec, language="en", temperature=0.0, condition_on_previous_text=True,
                                      initial_prompt=prompt, word_timestamps=True, vad=False, suppress_silence=True,
                                      suppress_ts_tokens=True, regroup=False, verbose=None, fp16=False,
                                      ignore_compatibility=True, sample_len=16)
        da, db = got.to_dict(), theirs.to_dict()
        assert len(da["segments"]) >= 1
        _assert_same(da, db, REL)


def test_languages_never_share_a_decode_batch(env, monkeypatch):
    """A multilingual model with a per-recording language list, one of them detected: every round runs one language, every
    result equals the per-recording call with that recording's language, and the detected language is the one
    ``detect_language_of`` finds for the recording alone."""
    import stable_ts_b200.transcribe as T
    stand, recs = env["stand_ml"], env["recs"]
    langs = ["en", "de", None, "en"]
    owner = {r.untyped_storage().data_ptr(): k for k, r in enumerate(recs)}
    rounds = []
    real = T.transcribe_windows

    def spy(model, tokenizer, audios, **kw):
        rounds.append((tokenizer.language, [owner[a.untyped_storage().data_ptr()] for a in audios]))
        return real(model, tokenizer, audios, **kw)
    kw = dict(KW, batch_windows=16, shard_seconds=30.0)
    monkeypatch.setattr(T, "transcribe_windows", spy)
    batch = stand.transcribe_batch(recs, language=langs, initial_prompt=PROMPTS, **kw)
    monkeypatch.setattr(T, "transcribe_windows", real)
    detected = stand.detect_language_of(recs[2][:480000])
    want = [lang or detected for lang in langs]
    assert [r.to_dict()["language"] for r in batch] == want
    assert rounds and any(len(ks) > 1 for _, ks in rounds)
    for lang, ks in rounds:
        assert all(want[k] == lang for k in ks), (lang, ks)
    for rec, lang, prompt, got in zip(recs, langs, PROMPTS, batch):
        alone = stand.transcribe(rec, language=lang, initial_prompt=prompt, **kw).to_dict()
        assert alone["language"] == got.to_dict()["language"]
        _assert_same(got.to_dict(), alone, REL)


def test_argument_errors(env):
    from stable_ts_b200.tokenizer import get_tokenizer
    stand, recs = env["stand"], env["recs"][:2]
    assert stand.transcribe_batch([], language="en") == []
    with pytest.raises(ValueError):
        stand.transcribe_batch(recs, language=["en"])
    with pytest.raises(ValueError):
        stand.transcribe_batch(recs, language="en", initial_prompt=["a", "b", "c"])
    with pytest.raises(TypeError):
        stand.transcribe_batch(recs, language="en", clip_timestamps=[0.0, 5.0])
    tk = get_tokenizer(stand, language="en", task="transcribe", synthetic=True)
    with pytest.raises(ValueError):
        stand.transcribe_batch(recs, language=["en", "en"], tokenizer=tk)
    with pytest.raises(NotImplementedError):
        stand.transcribe_batch(recs, language="en", beam_size=5)
    with pytest.raises(TypeError):
        stand.transcribe_batch(recs, language="en", vad=True)
