"""Two models of one process, on two devices, give the same results.

Function attributes (the opt-in to more than the default dynamic shared memory) and SM counts belong to a device, so a
model on a second device must not rely on what the first device was configured with.  The decode-step linears take the
batched GEMV at B <= 16 (88 KB of dynamic shared memory for fc2, whose K >= 1280) and the cluster linear at B = 17..128."""
import pytest
import torch

pytestmark = pytest.mark.gpu
STEPS = 32


def _transcribe(device, B):
    from oracle import stable_path as SP
    from stable_ts_b200.api import load_model
    from stable_ts_b200.decode import DecodingOptions
    from stable_ts_b200.tokenizer import get_tokenizer
    from stable_ts_b200.transcribe import transcribe_windows
    model = load_model("tiny", device=device, seed=0, allow_random=True)
    tk = get_tokenizer(model, language="en", task="transcribe", synthetic=True)
    audio = torch.stack([SP.synth_audio(480000, seed=3000 + i) for i in range(B)])
    script = torch.tensor([SP.synth_token_script(STEPS, tk.eot, seed=4321 + i) for i in range(B)], dtype=torch.int32)
    segs, info = transcribe_windows(model, tk, audio, forced_tokens=script.T.contiguous(),
                                    options=DecodingOptions(language="en", sample_len=STEPS, max_initial_timestamp=None))
    words = [[(w["word"], w["tokens"], w["start"], w["end"], w["probability"]) for s in ws for w in s["words"]] for ws in segs]
    return torch.as_tensor(info["step_argmax"]).cpu(), words


@pytest.mark.parametrize("B", [2, 24])
def test_second_device_matches_the_first(B):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    argmax0, words0 = _transcribe("cuda:0", B)
    argmax1, words1 = _transcribe("cuda:1", B)
    assert argmax0.shape[1] == B
    assert torch.equal(argmax0, argmax1)
    assert sum(len(w) for w in words0) > 0
    assert words0 == words1
