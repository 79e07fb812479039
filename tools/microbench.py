"""Developer micro-benchmarks of single kernels through the C ABI (CUDA-event timed, cold weights: the working set of
rotating weight copies exceeds the 126 MB L2 so every launch streams its weights from HBM, as in a real decode step).

    python tools/microbench.py gemv      # decode-step linear shapes of large-v3 at 16 / 64 sequences
    python tools/microbench.py dtw       # DTW at 16 / 64 windows x [101 x 1500]
    python tools/microbench.py step 120 4   # ms per decode step (120 windows, 4 decoder layers of large-v3 width)
    python tools/microbench.py attention # encoder attention (stb_attention) at 48 windows x 20 heads x 1500 x 1500
    python tools/microbench.py gemm      # stb_gemm at the encoder / forced-decoder shapes of 48 large-v3 windows
"""
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stable_ts_b200 import _lib as L  # noqa: E402


def _time(fn, iters, graph=True):
    """us per call; the calls are captured into one CUDA graph (no Python / ctypes launch overhead in the timing)"""
    for i in range(3):
        fn(i)
    torch.cuda.synchronize()
    if graph:
        st = torch.cuda.Stream()
        with torch.cuda.stream(st):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=st):
                for i in range(iters):
                    fn(i)
        g.replay()
        torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 5 if graph else 1
    e0.record()
    for _ in range(reps):
        if graph:
            g.replay()
        else:
            for i in range(iters):
                fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (iters * reps) * 1e3      # us


def bench_gemv(batches=(16, 64), shapes=((1280, 1280), (3840, 1280), (5120, 1280), (1280, 5120), (51866, 1280)), iters=200):
    lib = L.lib()
    out = []
    for Bn in batches:
        for (N, K) in shapes:
            copies = max(2, int(300e6 // (N * K * 4)) + 1)
            wh = torch.randn(copies, N, K, device="cuda").half()
            wl = torch.randn(copies, N, K, device="cuda").half() * 1e-3
            xh = torch.randn(Bn, K, device="cuda").half()
            xl = torch.randn(Bn, K, device="cuda").half() * 1e-3
            ld = (N + 7) // 8 * 8
            o = torch.empty(Bn, ld, device="cuda")

            def run(i):
                c = i % copies
                L.check(lib.stb_gemv(L.ptr(xh), L.ptr(xl), Bn, K, L.ptr(wh[c]), L.ptr(wl[c]), N, None, 0, None, 0, L.ptr(o),
                                     None, None, ld, L.stream_ptr()))
            us = _time(run, min(iters, 40))
            gbs = N * K * 4 / us / 1e3
            out.append(dict(B=Bn, N=N, K=K, us=round(us, 2), weight_GBps=round(gbs, 1)))
            print(out[-1], flush=True)
            del wh, wl
    return out


def bench_dtw(batches=(16, 64, 148)):
    lib = L.lib()
    out = []
    for Bn in batches:
        R, F = 101, 1500
        x = torch.randn(Bn, R, F, device="cuda")
        jumps = torch.zeros(Bn, R, dtype=torch.int32, device="cuda")
        ws = torch.empty(lib.stb_dtw_ws_bytes(Bn, R, F), dtype=torch.uint8, device="cuda")

        def run(i):
            L.check(lib.stb_dtw(L.ptr(x), Bn, R, F, F, 1, L.ptr(jumps), None, None, L.ptr(ws), ws.numel(), L.stream_ptr()))
        us = _time(run, 50)
        out.append(dict(windows=Bn, R=R, F=F, us=round(us, 1)))
        print(out[-1], flush=True)
    return out


def _card():
    """name, power limit and max SM clock of the current device, read next to the measurement they qualify"""
    import subprocess
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    # nvidia-smi numbers the cards in PCI order, whatever CUDA_VISIBLE_DEVICES makes of them: select by PCI address
    pci = f"{p.pci_domain_id:08X}:{p.pci_bus_id:02X}:{p.pci_device_id:02X}.0"
    info = {"name": p.name, "pci_bus_id": pci}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={pci}", "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.strip()
        pl, mhz = (v.strip() for v in q.split(","))
        info.update(power_limit_w=float(pl), sm_max_mhz=int(mhz))
    except Exception as e:
        info["nvidia_smi"] = f"unavailable: {e}"
    return info


def bench_attention(windows=48, heads=20, T=1500, iters=10):
    """stb_attention at the encoder's shape (large-v3: 20 heads of 64, 1500 x 1500, one launch per layer for all windows).
    Algorithmic work is 4 T^2 64 per (window, head); executed work counts the fp16 passes of every product (3 in parity
    mode, 1 in fp16 mode).  The peak is the H100 SXM data sheet's dense fp16 rate, not a measured one."""
    lib = L.lib()
    d, ldk = 64 * heads, (T + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(windows, T, 2 * d, device="cuda", generator=g)           # q | k, as the encoder's fused projection
    vT = torch.zeros(windows, heads, 64, ldk, device="cuda")
    vT[..., :T] = torch.randn(windows, heads, 64, T, device="cuda", generator=g)
    xh, vh = x.half(), vT.half()
    xl, vl = (x - xh.float()).half(), (vT - vh.float()).half()
    del x, vT
    out_hi = torch.empty(windows, T, d, dtype=torch.float16, device="cuda")
    out_lo = torch.empty_like(out_hi)
    flop = 4.0 * T * T * 64 * heads * windows
    res = {"card": _card(), "shape": dict(windows=windows, heads=heads, Mq=T, Mk=T), "algorithmic_gflop_per_launch": flop / 1e9,
           "peak_tflops": 989.0, "peak_source": "H100 SXM data sheet, dense fp16 at 700 W (not measured)", "runs": []}
    for passes in (3, 1):
        lo = passes == 3
        oq = L.Operand(L.ptr(xh), L.ptr(xl) if lo else None, T, 64, 2 * d, 64, T * 2 * d)
        ok = L.Operand(L.ptr(xh[..., d:]), L.ptr(xl[..., d:]) if lo else None, T, 64, 2 * d, 64, T * 2 * d)
        ov = L.Operand(L.ptr(vh), L.ptr(vl) if lo else None, 64, ldk, ldk, 64 * ldk, d * ldk)

        def run(i):
            L.check(lib.stb_attention(ctypes.byref(oq), ctypes.byref(ok), ctypes.byref(ov), windows, heads, T, T,
                                      L.ptr(out_hi), L.ptr(out_lo) if lo else None, d, 64, T * d, L.stream_ptr()))
        us = _time(run, iters)
        alg = flop / (us * 1e-6) / 1e12
        res["runs"].append(dict(passes=passes, us_per_launch=round(us, 1), algorithmic_tflops=round(alg, 1),
                                executed_tflops=round(alg * passes, 1), executed_frac_of_peak=round(alg * passes / 989.0, 3)))
        print(res["runs"][-1], flush=True)
    print(res["card"], flush=True)
    return res


def bench_gemm(windows=48, iters=6):
    """stb_gemm at the shapes one large-v3 step runs (48 windows of 1500 encoder rows, a forced decode of 229 rows per
    window), split-fp16 operands (3 passes).  Executed TFLOP/s counts the 3 passes; the peak is the H100 SXM data
    sheet's dense fp16 rate, not a measured one."""
    lib = L.lib()
    T, F, d, Tp, H = 1500, 3000, 1280, 1504, 20
    M, Md = windows * T, windows * 229
    g = torch.Generator(device="cuda").manual_seed(0)

    def split(*shape, scale=1.0):
        x = torch.randn(*shape, device="cuda", generator=g) * scale
        h = x.half()
        return h, (x - h.float()).half()

    def zeros(n, dt=torch.float16):
        return torch.zeros(n, dtype=dt, device="cuda")

    res = {"card": _card(), "windows": windows, "peak_tflops": 989.0,
           "peak_source": "H100 SXM data sheet, dense fp16 at 700 W (not measured)", "runs": []}
    xh, xl = split(M, 4 * d)                 # large enough for every A operand below (fc2's K = 5120)
    wh, wl = split(51866, d, scale=0.03)     # large enough for every weight below (logits' 51866 rows)
    bias = torch.randn(51866, device="cuda", generator=g)
    out_h, out_l = zeros(M * 4 * d), zeros(M * 4 * d)
    out_f = zeros(max(M * d, Md * 51872), torch.float32)

    def op(hi, lo, rows, k, rs, hs=0, bs=0):
        return L.Operand(L.ptr(hi), L.ptr(lo), rows, k, rs, hs, bs)

    def ep(ld, split_out=True, f32=False, res_=False, act=0, bias_=True, transposed=False, out_h_stride=0, out_b=0,
           res_b=None):
        e = L.Epilogue()
        if split_out:
            e.out_hi, e.out_lo = L.ptr(out_h), L.ptr(out_l)
        if f32:
            e.out_f32 = L.ptr(out_f)
        e.ld_out, e.out_h_stride, e.out_b_stride, e.transposed = ld, out_h_stride, out_b, int(transposed)
        e.bias = L.ptr(bias) if bias_ else None
        if res_:
            e.residual, e.ld_res = L.ptr(out_f), ld
            e.res_b_stride = out_b if res_b is None else res_b
        e.alpha, e.act = 1.0, act
        return e

    A1280 = op(xh, xl, M, d, d)
    Ab = op(xh, xl, T, d, d, 0, T * d)                     # per-window view (batch stride T rows)
    cases = [
        ("enc q|k", A1280, op(wh, wl, 2 * d, d, d), 1, 1, ep(2 * d), M, 2 * d, d),
        ("enc V^T", Ab, op(wh, wl, d, d, d), windows, 1, ep(Tp, transposed=True, out_b=d * Tp), M, d, d),
        ("enc out", A1280, op(wh, wl, d, d, d), 1, 1, ep(d, split_out=False, f32=True, res_=True), M, d, d),
        ("enc fc1", A1280, op(wh, wl, 4 * d, d, d), 1, 1, ep(4 * d, act=1), M, 4 * d, d),
        ("enc fc2", op(xh, xl, M, 4 * d, 4 * d), op(wh, wl, d, 4 * d, 4 * d), 1, 1,
         ep(d, split_out=False, f32=True, res_=True), M, d, 4 * d),
        ("enc conv2", op(xh, xl, T, 3 * d, 2 * d, 0, (F + 2) * d), op(wh, wl, d, 3 * d, 3 * d), windows, 1,
         ep(d, split_out=False, f32=True, res_=True, act=1, out_b=T * d, res_b=0), M, d, 3 * d),
        ("cross K per-head", Ab, op(wh, wl, 64, d, d, 64 * d, 0), windows, H,
         ep(64, bias_=False, out_h_stride=T * 64, out_b=H * T * 64), M, d, d),
        ("dec fc1", op(xh, xl, Md, d, d), op(wh, wl, 4 * d, d, d), 1, 1, ep(4 * d, act=1), Md, 4 * d, d),
        ("dec logits", op(xh, xl, Md, d, d), op(wh, wl, 51866, d, d), 1, 1,
         ep(51872, split_out=False, f32=True, bias_=False), Md, 51866, d),
    ]
    if any(f == "head_cols" for f, _ in L.Epilogue._fields_):
        e = ep(64, bias_=False, out_h_stride=T * 64, out_b=H * T * 64)
        e.head_cols = 64
        cases.insert(7, ("cross K head-major", Ab, op(wh, wl, d, d, d), windows, 1, e, M, d, d))
    for name, a, b, nb, nh, e, m, n, k in cases:
        def run(i, a=a, b=b, nb=nb, nh=nh, e=e):
            L.check(lib.stb_gemm(ctypes.byref(a), ctypes.byref(b), nb, nh, ctypes.byref(e), L.stream_ptr()))
        us = _time(run, iters)
        tf = 3 * 2.0 * m * n * k / (us * 1e-6) / 1e12
        res["runs"].append(dict(shape=name, M=m, N=n, K=k, us=round(us, 1), executed_tflops=round(tf, 1),
                                executed_frac_of_peak=round(tf / 989.0, 3)))
        print(res["runs"][-1], flush=True)
    print(res["card"], flush=True)
    return res


def bench_step(windows=120, layers=4, s1=24, s2=72):
    """ms per KV-cached decode step of a large-v3-WIDTH model with `layers` decoder layers (cross K/V of 120 windows x 32
    layers would not leave room for A/B runs), from the slope between two forced decodes of s1 and s2 steps (graph replay):
    microbench.py step [windows] [layers]"""
    import time
    from stable_ts_b200.api import random_state_dict
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    from stable_ts_b200.model import B200Whisper
    from stable_ts_b200.tokenizer import get_tokenizer
    from oracle.whisper_ref.model import ModelDimensions      # dims container only (tools/ is developer tooling)
    dims = ModelDimensions(128, 1500, 1280, 20, 1, 51866, 448, 1280, 20, layers)
    model = B200Whisper(dims, random_state_dict(dims, 0), device="cuda")
    tk = get_tokenizer(model, language="en", task="transcribe", synthetic=True)
    g = torch.Generator().manual_seed(0)
    audio = (torch.randn(windows, 480000, generator=g) * 0.1).cuda()
    enc = model.encode(model.log_mel(audio))
    forced = torch.randint(300, 50000, (s2, windows), generator=g, dtype=torch.int32)

    def run(steps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        decode_windows(model, tk, enc, DecodingOptions(language="en", sample_len=steps), forced_tokens=forced[:steps],
                       reuse_buffers=True)
        torch.cuda.synchronize()
        return (time.perf_counter() - t) * 1e3
    run(s1)
    a = min(run(s1) for _ in range(3))
    b = min(run(s2) for _ in range(3))
    per_step = (b - a) / (s2 - s1)
    L.lib().stb_prof_enable(1)
    decode_windows(model, tk, enc, DecodingOptions(language="en", sample_len=8), forced_tokens=forced[:8], use_graph=False,
                   reuse_buffers=True)
    prof = L.prof_report()
    L.lib().stb_prof_enable(0)
    table = {k: {"n": v["n"], "us_avg": round(v["ms"] * 1e3 / max(v["n"], 1), 2)} for k, v in prof.items()}
    out = dict(windows=windows, layers=layers, ms_per_step=round(per_step, 3), ms_per_layer_step=round(per_step / layers, 4),
               fixed_ms=round(a - per_step * s1, 1), eager_kernels=table)
    print(out, flush=True)
    return out


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "gemv"
    if what == "step":
        res = bench_step(*(int(v) for v in sys.argv[2:4]))
    elif what == "ncu":          # short run for `ncu -k regex:...`: fc1 / fc2 at 64 sequences + one DTW batch
        res = [bench_gemv((64,), ((5120, 1280), (1280, 5120)), iters=4), bench_dtw((16,))]
    else:
        res = {"gemv": bench_gemv, "dtw": bench_dtw, "attention": bench_attention, "gemm": bench_gemm}[what]()
    print(json.dumps({what: res, "env": {k: v for k, v in os.environ.items() if k.startswith("STB_")}}))
