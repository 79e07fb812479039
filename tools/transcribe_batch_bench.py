"""Throughput of ``model.transcribe_batch`` against a loop of ``model.transcribe`` over many short recordings.

    python tools/transcribe_batch_bench.py [--clips 96] [--reps 3] [--out result.json]

Workload: large-v3 with seeded random weights, ``--clips`` seeded synthetic clips of 4-28 s (one window each),
``temperature=0.0`` and ``sample_len=64`` so that random-weight decoding has a bounded length.  Arms: the loop (every clip
decoded at batch 1) and ``transcribe_batch`` at ``batch_windows`` 16 and 48.  Every arm runs once as a warm-up, then the arms
alternate for ``--reps`` repetitions; each repetition's wall clock ends in ``torch.cuda.synchronize()``.  Reported per arm:
clips/s and audio-seconds/s (median repetition), kernel launches per repetition (library launches + CUDA-graph replays),
and peak HBM.  The device name, power limit and SM clocks are read in the same run.  The batched arms must reproduce the
loop's tokens and word times: the script writes its result and then fails if one does not.  ``segments`` / ``words``
in the result say how much output that comparison covered: with random weights the kept text can be empty."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import stable_path as SP  # noqa: E402
from stable_ts_b200 import _lib as L  # noqa: E402
from stable_ts_b200 import load_model  # noqa: E402

SR = 16000
# no_speech_threshold=None: no window is skipped on its no-speech probability, so every window is decoded in every arm
KW = dict(language="en", temperature=0.0, sample_len=64, regroup=False, no_speech_threshold=None)


def _card():
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    pci = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
    info = {"name": p.name, "pci_bus_id": pci}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={pci}", "--query-gpu=power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
        pl, mx, sm = (v.strip() for v in q.split(","))
        info.update(power_limit_w=float(pl), sm_max_mhz=int(mx), sm_mhz_after=int(sm))
    except Exception as e:                                   # the timings still stand; say what is missing
        info["nvidia_smi_error"] = repr(e)
    return info


def clips(n: int):
    g = torch.Generator().manual_seed(2026)
    lengths = (torch.randint(4 * SR, 28 * SR + 1, (n,), generator=g)).tolist()
    return [SP.synth_audio(int(m), seed=1000 + k) for k, m in enumerate(lengths)]


def tokens_of(results):
    """tokens and word times of every segment of every clip"""
    return [[(s["tokens"], [(w["start"], w["end"]) for w in s["words"]]) for s in r.to_dict()["segments"]] for r in results]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=96)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transcribe_batch_bench needs a CUDA device")
    torch.cuda.set_device(0)
    model = load_model(args.model, device="cuda:0", allow_random=True)
    audio = clips(args.clips)
    audio_s = sum(a.numel() for a in audio) / SR
    arms = {
        "loop": lambda: [model.transcribe(a, **KW) for a in audio],
        "batch16": lambda: model.transcribe_batch(audio, batch_windows=16, **KW),
        "batch48": lambda: model.transcribe_batch(audio, batch_windows=48, **KW),
    }
    lib = L.lib()
    stats = {k: dict(s=[], launches=[], peak_bytes=0) for k in arms}
    ref, mismatch = None, set()
    for rep in range(args.reps + 1):                         # repetition 0 warms every arm up and is not reported
        for name, run in arms.items():
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            l0 = lib.stb_launch_count() + model.graph_kernel_launches
            t0 = time.perf_counter()
            out = run()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            toks = tokens_of(out)
            if ref is None:
                ref = toks
            if toks != ref:
                mismatch.add(name)
            if rep:
                st = stats[name]
                st["s"].append(dt)
                st["launches"].append(int(lib.stb_launch_count() + model.graph_kernel_launches - l0))
                st["peak_bytes"] = max(st["peak_bytes"], int(torch.cuda.max_memory_allocated()))
            print(f"[transcribe_batch_bench] rep {rep} {name}: {dt:.2f} s", file=sys.stderr)
    res = dict(model=args.model, clips=args.clips, audio_s=round(audio_s, 2), reps=args.reps, options=KW,
               segments=sum(len(r) for r in ref), words=sum(len(w) for r in ref for _, w in r), arms={})
    for name, st in stats.items():
        s = statistics.median(st["s"])
        res["arms"][name] = dict(s_median=round(s, 3), s_all=[round(v, 3) for v in st["s"]],
                                 clips_per_s=round(args.clips / s, 2), audio_s_per_s=round(audio_s / s, 1),
                                 launches_per_rep=statistics.median(st["launches"]),
                                 peak_hbm_gb=round(st["peak_bytes"] / 1e9, 2))
    res["tokens_equal_loop"] = {name: name not in mismatch for name in arms}
    res["card"] = _card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    assert not mismatch, f"tokens or word times differ from the loop's: {sorted(mismatch)}"


if __name__ == "__main__":
    main()
