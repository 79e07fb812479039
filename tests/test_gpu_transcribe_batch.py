"""GPU tests of ``model.transcribe_batch``: recordings of different lengths (one of two shards, one with a silent gap, one all
zeros, one shorter than a token, one given as a WAV path) through shared device batches give every recording what
``model.transcribe`` gives it alone.  The encoder and the teacher-forced decoder compute every row independently of the batch,
so detected languages, tokens, seeks and times are identical; word probabilities may move by the decode-step route the batch
size selects (above 16 sequences the cluster route replaces the GEMV route), bounded as in tests/test_gpu_depth.py."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
SR = 16000
KW = dict(regroup=False, sample_len=24, temperature=0.0)


def _gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


_MODELS = {}


def _model(name):
    if name not in _MODELS:
        from stable_ts_b200 import load_model
        _MODELS[name] = load_model(name, device="cuda:0", allow_random=True)
    return _MODELS[name]


def _recordings(tmp_path):
    """4 s, 29.5 s, 47 s (two shards), 75 s with a 5 s silent gap, 10 s of zeros, and 12.5 s as a 16-bit WAV file."""
    from oracle import stable_path as SP
    from oracle.audio_io import make_wav
    wav = (SP.synth_audio(200000, seed=46).numpy() * 32767).astype(np.int16)
    path = tmp_path / "clip.wav"
    path.write_bytes(make_wav(wav, SR, 1))
    return [SP.synth_audio(64000, seed=41), SP.synth_audio(472000, seed=42), SP.synth_gapped_audio(752000, seed=43),
            torch.cat([SP.synth_audio(560000, seed=44), torch.zeros(80000), SP.synth_audio(560000, seed=45)]),
            torch.zeros(160000), str(path)]


def _compare(da, db):
    """-> the largest relative word-probability difference; everything else must be identical."""
    assert da["language"] == db["language"] and len(da["segments"]) == len(db["segments"])
    worst = 0.0
    for sa, sb in zip(da["segments"], db["segments"]):
        for k in ("id", "seek", "start", "end", "text", "tokens"):
            assert sa.get(k) == sb.get(k), k
        assert len(sa["words"]) == len(sb["words"])
        for wa, wb in zip(sa["words"], sb["words"]):
            assert (wa["word"], wa["tokens"], wa["start"], wa["end"]) == (wb["word"], wb["tokens"], wb["start"], wb["end"])
            worst = max(worst, abs(wa["probability"] - wb["probability"]) / max(abs(wb["probability"]), 1e-30))
    return worst


def test_batched_language_detection_equals_single(tmp_path):
    _gpu()
    from stable_ts_b200.api import _as_waveform
    gm = _model("tiny")
    recs = _recordings(tmp_path)
    res = gm.transcribe_batch(recs, language=None, batch_windows=4, **KW)
    alone = [gm.detect_language_of(_as_waveform(r, gm)[:480000]) for r in recs]
    print("languages:", alone)
    assert [r.to_dict()["language"] for r in res] == alone


@pytest.mark.parametrize("name", ["tiny", "tiny.en"])
@pytest.mark.parametrize("batch_windows", [2, 16, 48])
def test_batch_equals_separate_calls(tmp_path, name, batch_windows):
    _gpu()
    gm = _model(name)
    recs = _recordings(tmp_path)
    kw = dict(KW, batch_windows=batch_windows)
    batch = gm.transcribe_batch(recs, language=None, **kw)
    worst, n_words = 0.0, 0
    for rec, got in zip(recs, batch):
        da, db = got.to_dict(), gm.transcribe(rec, language=None, **kw).to_dict()
        worst = max(worst, _compare(da, db))
        n_words += sum(len(s["words"]) for s in da["segments"])
    print(f"{name} batch_windows={batch_windows}: {n_words} words, largest word-probability difference {worst:.2e} relative")
    assert n_words > 0 and worst <= 2e-3


def test_only_voice_freq_in_a_batch_equals_filtering_first(tmp_path):
    _gpu()
    from stable_ts_b200.api import _as_waveform
    from stable_ts_b200.audio_io import voice_freq_filter
    gm = _model("tiny")
    recs = _recordings(tmp_path)
    hum = [r + 0.2 * torch.sin(2 * np.pi * 60 * torch.arange(r.numel()) / SR) for r in recs[:4]]   # mains hum below the band
    recs = hum + recs[4:]
    a = gm.transcribe_batch(recs, language=None, only_voice_freq=True, batch_windows=16, **KW)
    b = gm.transcribe_batch([voice_freq_filter(_as_waveform(r, gm).cuda()) for r in recs], language=None, batch_windows=16,
                            **KW)
    assert [x.to_dict() for x in a] == [y.to_dict() for y in b]
    assert any(x.to_dict()["segments"] for x in a)


@pytest.mark.parametrize("name", ["tiny", "tiny.en"])
def test_silent_and_tiny_recordings_come_back_empty(name):
    _gpu()
    from oracle import stable_path as SP
    gm = _model(name)
    # 10 s of zeros, and 200 samples: less than one 320-sample token, the half-frame that the alignment pass still needs
    recs = [SP.synth_audio(300000, seed=51), torch.zeros(160000), SP.synth_audio(200, seed=52), SP.synth_audio(90000, seed=53)]
    batch = gm.transcribe_batch(recs, language=None, batch_windows=16, **KW)
    for k in (1, 2):
        assert batch[k].to_dict()["segments"] == []
    for rec, got in zip(recs, batch):
        _compare(got.to_dict(), gm.transcribe(rec, language=None, batch_windows=16, **KW).to_dict())
