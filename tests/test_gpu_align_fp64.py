"""GPU tests of both ends of the word-alignment path against float64 references computed on the CPU: the attention-matrix
post-processing in its three variants (csrc/qkpost.cu), the token probabilities (token_prob_kernel and
softmax_probs_kernel, csrc/elementwise.cu) and the log-mel front end (csrc/logmel.cu, model.log_mel).

- stb_qk_postprocess (legacy alignment heads): F = 1..1504 (the filter is off at F <= 3; F = 4..7 reflects on both sides
  of one window; 1504 = QK_MAXV x 32), R = 1 / 2 / 109, S = 0 / 1 / 3 with S = 0 and R = M, A = 1 / 10, qk_scale 0.7 / 1 /
  1.9, medfilt_width 7 / 1.  R = 1 (and F = 1) is 0 / 0: NaN at exactly the same elements.  One case holds every one of
  the 5040 orderings of 7 consecutive pre-median values, so the sorting network of median7 is checked exhaustively; one
  case has near-constant columns.
- stb_qk_postprocess_dynamic: 24 / 144 / 640 / 1280 heads, 1 / 6 / 20 heads per token, the first iteration (argmax peak)
  and a given prev_jumps (repeated values, last midpoint reaching F) with reuse_softmax; the best heads are planted at
  indices on both sides of the 64-bit words of the selection mask, in a different order for every token row.
- stb_qk_postprocess_new: the same head counts with planted heads, top-k 1 / 20, the four weightings of the head score
  (one where the coverage penalty changes the top-k set), qk_scale != 1 and medfilt_width 1.
- stb_token_probs, stb_softmax_probs: 50257 classes at a pitch of 51872, targets at 0, n - 1, the row maximum and a -1e4
  logit, quantized rows with many ties (the rank bitwise), all-equal rows (bitwise fp32(1 / n)).
- stb_logmel and model.log_mel: align mode (n = 1 .. 480000, per-window maximum) and refine mode (n = 201 .. 480000,
  maximum over the batch, a partial last CTA), 80 and 128 mels; speech, tones on and between bins, a clipped square, DC
  plus noise, 1e-5 noise, impulses at both reflect edges and an all-zero window (exactly -1.5).
- Bitwise invariants: inputs the kernels must not read hold NaN (legacy qk rows outside [S, S+R) and columns >= F, logit
  columns >= n_classes, audio past n_samples) or, for the dynamic and new paths that turn scores into head indices, the
  finite +3e4 (qk columns >= F); a NaN-filled legacy / log-mel workspace gives the same output as a zeroed one; output
  pad columns keep a sentinel; item b of a batch is bitwise the item run alone.

The references restate the stable-ts formulas in float64 (stable_whisper/timing.py:85-110 for the legacy and dynamic
heads, :115-163 for the new aligner; whisper.timing.median_filter; whisper.audio.log_mel_spectrogram) and are fed the
same fp32 inputs as the kernels.  Where a z-norm divides by a column's std, or a log divides by a mel power, the error
grows with a condition number kappa, so those outputs are gated per element by |err| <= a kappa + b: a bounds
|err| / kappa over all elements, b the error where kappa <= 10.  The bounds are 1.25x the worst error measured on an
NVIDIA H100 80GB HBM3 at 700 W, rounded up to two digits; the measured worsts are next to each bound.

Run on an H100:  python -m pytest tests/test_gpu_align_fp64.py -q -s
"""
import functools

import numpy as np
import pytest
import torch
from numpy.lib.stride_tricks import sliding_window_view

pytestmark = pytest.mark.gpu

NAN = float("nan")
SENTINEL = -7.25                  # pre-filled into output pad columns
POISON = 3.0e4                    # unread qk columns of the dynamic / new paths (finite: those paths turn scores into indices)
LDQ = 1508                        # qk row pitch: at least 4 unread columns after F = 1504

# bounds: 1.25x the worst error measured on an NVIDIA H100 80GB HBM3 at 700 W, rounded up to two digits
LEGACY_A = 5.5e-7                 # legacy: |err| / kappa over all elements: worst 4.36e-7 (near-constant columns)
LEGACY_B = 6.0e-7                 # legacy: |err| where kappa <= 10: worst 4.79e-7
DYN_A = 7.6e-7                    # dynamic heads: |err| / kappa: worst 6.08e-7
DYN_B = 4.9e-6                    # dynamic heads: |err| where kappa <= 10: worst 3.90e-6
NEW_BOUND = 1.8e-6                # new aligner, |err| / |ref| per element: worst 1.38e-6
PROB_BOUND = 5.2e-7               # token probability, |err| / max(p, 2^-126): worst 4.15e-7
SOFTMAX_BOUND = 2.7e-7            # softmax_probs per row, relative to the row's largest probability: worst 2.15e-7
MEL_A = 3.6e-6                    # log-mel |err| / kappa: worst 2.87e-6
MEL_B = 5.4e-6                    # log-mel |err| where kappa <= 10: worst 4.29e-6 (128 mels)

# heads planted as the best ones: both sides of every 64-bit word boundary of the selection mask in use up to 1280 heads
PLANT = (5, 63, 64, 127, 128, 639, 1279)


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from stable_ts_b200 import _lib
    _lib.lib()
    name = torch.cuda.get_device_name()
    try:
        import subprocess
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                         # nvidia-smi missing: the card name alone
        pl = "unknown"
    print(f"\ndevice: {name}, power limit {pl}")
    return _lib


def _bits(t):
    """bit pattern of a float32 tensor / array (bitwise comparisons that NaN cannot spoil)"""
    return torch.as_tensor(t).contiguous().view(torch.int32)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _softmax(x):
    """float64 softmax over the last axis"""
    e = np.exp(x - x.max(-1, keepdims=True))
    return e / e.sum(-1, keepdims=True)


def _taps(x, fn):
    """fn over the 7 reflect-padded neighbours of every column of x [..., F] (whisper.timing.median_filter pads with
    mode="reflect", no edge repeat), in row chunks so that the 7x copy stays small"""
    F = x.shape[-1]
    flat = x.reshape(-1, F)
    out = np.empty_like(flat)
    for i in range(0, flat.shape[0], 1024):
        xp = np.pad(flat[i:i + 1024], ((0, 0), (3, 3)), mode="reflect")
        out[i:i + 1024] = fn(sliding_window_view(xp, 7, axis=-1))
    return out.reshape(x.shape)


def _median(x, width):
    """whisper.timing.median_filter: off for width 1 and when F <= width // 2"""
    if width == 1 or x.shape[-1] <= 3:
        return x
    return _taps(x, lambda w: np.partition(w, 3, axis=-1)[..., 3])


def _znorm_median_mean(W, width):
    """timing.py:108-110 and the head mean of :194 on W [B][A][R][F] float64 -> (matrix [B][R][F], kappa [B][F]).
    kappa of an output column = max over heads and the window's columns of max_r |W[r, c]| / std_c."""
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = W.mean(-2, keepdims=True)
        std = np.sqrt(((W - mean) ** 2).mean(-2, keepdims=True))
        Z = (W - mean) / std
        kap = np.abs(W).max(-2) / std[..., 0, :]                 # [B][A][F]
    if width == 7 and W.shape[-1] > 3:
        kap = _taps(kap, lambda w: w.max(-1))
    return _median(Z, width).mean(1), kap.max(1), Z


def _gate(name, out, ref, kap, A_bound, B_bound):
    """NaN at the same elements; then |err| <= a kappa + b.  Returns (worst |err| / kappa, worst |err| at kappa <= 10)."""
    out = out.astype(np.float64)
    nan_o, nan_r = np.isnan(out), np.isnan(ref)
    assert np.array_equal(nan_o, nan_r), f"{name}: NaN at {int((nan_o != nan_r).sum())} elements where float64 differs"
    fin = ~nan_r
    if not fin.any():
        print(f"{name}: all NaN, as in float64")
        return 0.0, 0.0
    k = np.broadcast_to(kap, ref.shape)[fin]
    err = np.abs(out[fin] - ref[fin])
    a = float((err / np.maximum(k, 1e-300)).max())
    low = k <= 10
    b = float(err[low].max()) if low.any() else 0.0
    print(f"{name}: worst |err| / kappa {a:.2e}, worst |err| at kappa <= 10 {b:.2e} (max kappa {k.max():.1e}, "
          f"max |err| {err.max():.2e})")
    assert (err <= A_bound * k + B_bound).all(), (name, a, b)
    assert b <= B_bound, (name, b)
    return a, b


# ---------------------------------------------------------------------------------------------------------------
# legacy alignment heads
# ---------------------------------------------------------------------------------------------------------------
def _legacy_call(L, qk, S, R, F, scale, width, ws_fill):
    """stb_qk_postprocess on qk fp32 [B][A][M][LDQ] into a sentinel-filled matrix with 4+ pad columns"""
    B, A, M, _ = qk.shape
    ldm = (F + 3) // 4 * 4 + 4
    lib = L.lib()
    out = torch.full((B, R, ldm), SENTINEL, device="cuda")
    ws = torch.full((lib.stb_qkpost_ws_bytes(B, A, R, F) // 4,), ws_fill, device="cuda")
    L.check(lib.stb_qk_postprocess(L.ptr(qk), B, A, M, LDQ, S, R, F, scale, width, L.ptr(out), ldm, L.ptr(ws),
                                   ws.numel() * 4, L.stream_ptr()))
    torch.cuda.synchronize()
    out = out.cpu()
    pad = out[..., F:]
    assert torch.equal(_bits(pad), _bits(torch.full_like(pad, SENTINEL))), "an output pad column was written"
    return out[..., :F]


def _count_orderings(Z):
    """number of distinct orderings among all windows of 7 consecutive columns of Z [..., F] (no reflection)"""
    seen = np.zeros(7 ** 7, dtype=bool)
    pw = 7 ** np.arange(7)
    flat = Z.reshape(-1, Z.shape[-1])
    for i in range(0, flat.shape[0], 512):
        w = sliding_window_view(flat[i:i + 512], 7, axis=-1).reshape(-1, 7)
        rank = np.argsort(np.argsort(w, axis=-1), axis=-1)
        seen[rank @ pw] = True
    return int(seen.sum())


LEGACY = [  # F, A, R, S, M (rows in memory), qk_scale, medfilt_width, kind
    (1, 10, 109, 1, 111, 1.0, 7, "random"),
    (2, 1, 2, 0, 2, 0.7, 7, "random"),          # S = 0, R = M
    (3, 10, 109, 3, 113, 1.9, 7, "random"),
    (4, 10, 2, 3, 6, 1.0, 7, "random"),
    (5, 1, 109, 0, 109, 0.7, 7, "random"),      # S = 0, R = M
    (7, 10, 1, 1, 3, 1.9, 7, "random"),         # R = 1: 0 / 0
    (8, 10, 109, 3, 113, 1.0, 1, "random"),
    (31, 1, 2, 1, 4, 1.9, 7, "random"),
    (32, 10, 109, 0, 109, 0.7, 7, "random"),
    (33, 10, 109, 3, 113, 1.0, 7, "random"),
    (937, 10, 109, 1, 111, 0.7, 7, "random"),
    (1500, 10, 109, 3, 113, 1.9, 7, "orderings"),
    (1500, 10, 109, 3, 113, 1.0, 1, "random"),
    (1500, 10, 109, 1, 111, 1.0, 7, "flat"),    # near-constant columns
    (1504, 10, 109, 0, 109, 1.0, 7, "random"),
    (1504, 1, 1, 3, 5, 0.7, 7, "random"),
]


@pytest.mark.parametrize("F,A,R,S,M,scale,width,kind", LEGACY)
def test_legacy_postprocess_matches_float64(L, F, A, R, S, M, scale, width, kind):
    """softmax(qk * scale) -> z-norm over the R rows (biased std) -> median -> head mean against float64, B = 3; qk rows
    outside [S, S+R) and columns >= F are NaN; a NaN-filled workspace gives the output of a zeroed one; item 1 alone
    gives item 1 of the batch."""
    B = 3
    g = np.random.default_rng(F * 1009 + R * 31 + A + S)
    if kind == "flat":                                        # every token row: one base row plus 1e-4 noise
        x = 3 * g.standard_normal((B, A, 1, F)) + 1e-4 * g.standard_normal((B, A, R, F))
    else:
        x = 3 * g.standard_normal((B, A, R, F))
    qk = np.full((B, A, M, LDQ), np.nan, np.float32)
    qk[:, :, S:S + R, :F] = x
    sc = float(np.float32(scale))
    ref, kap, Z = _znorm_median_mean(_softmax(qk[:, :, S:S + R, :F].astype(np.float64) * sc), width)
    qkd = _dev(qk)
    out = _legacy_call(L, qkd, S, R, F, scale, width, NAN)
    assert torch.equal(_bits(out), _bits(_legacy_call(L, qkd, S, R, F, scale, width, 0.0))), "depends on the workspace"
    assert torch.equal(_bits(out[1]), _bits(_legacy_call(L, qkd[1:2].contiguous(), S, R, F, scale, width, 0.0)[0])), \
        "item 1 alone differs from item 1 of the batch"
    _gate(f"legacy F={F} A={A} R={R} S={S} scale={scale} width={width} {kind}", out.numpy(), ref, kap[:, None, :],
          LEGACY_A, LEGACY_B)
    if kind == "orderings":
        n = _count_orderings(Z)
        print(f"legacy: {n} of 5040 orderings of 7 consecutive pre-median values")
        assert n == 5040


# ---------------------------------------------------------------------------------------------------------------
# dynamic heads and the new aligner: planted heads
# ---------------------------------------------------------------------------------------------------------------
def _planted(LH, n, seed):
    """n head indices: PLANT below LH first, then others spread over [0, LH)"""
    heads = [h for h in PLANT if h < LH]
    rest = [h for h in np.random.default_rng(seed).permutation(LH).tolist() if h not in heads]
    return heads + rest[:n - len(heads)]


def _bump(F, p, k, g):
    """a row peaked at column p with slope k over a floor of -20 plus noise (no softmax weight underflows in fp32, and no
    column is constant across rows)"""
    return np.maximum(3.0 - k * np.abs(np.arange(F) - p), -20.0 + 0.5 * g.standard_normal(F))


def _margin(v, n):
    """smallest relative gap between consecutive values among the first n + 1 of v sorted ascending, along the last axis"""
    s = np.sort(v, -1)[..., :n + 1]
    return float((np.diff(s, axis=-1) / np.abs(s[..., 1:])).min())


@functools.lru_cache(maxsize=1)
def _dyn_inputs(LH):
    """qk fp32 [B][LH][M][LDQ] for the dynamic heads: 21 planted heads per token row peak at the row's midpoint
    (floored) with slopes 2 * 0.8^j for rank j, in an order rotated by the row (the last row's rank-1 head is moved, see
    below); the other heads are diffuse with a +3 spike at a random column.  Rows outside [S, S+R) and columns >= F are +3e4.  -> (qk, prev_jumps [B][R], B, M, S, R, F)"""
    B, R, S, F = {24: (3, 40, 3, 1500), 144: (3, 29, 1, 937), 640: (2, 20, 3, 1500), 1280: (1, 20, 3, 1504)}[LH]
    M = S + R + 1
    g = np.random.default_rng(LH)
    jumps = np.sort(g.integers(0, F - 40, (B, R)), -1)
    jumps[:, 5] = jumps[:, 4]                                 # a repeated jump: zero-width interval
    jumps[:, -1] = F - 4                                      # the last midpoint, F - 2, is taken toward j1 = F
    nxt = np.concatenate([jumps[:, 1:], np.full((B, 1), F)], 1)
    mid = jumps + (nxt - jumps) * 0.5
    qk = np.full((B, LH, M, LDQ), POISON, np.float32)
    x = 0.5 * g.standard_normal((B, LH, R, F), dtype=np.float32)
    spike = g.integers(0, F, (B, LH, R))
    np.put_along_axis(x, spike[..., None], 3.0, axis=-1)
    planted = _planted(LH, 21, LH + 1)
    for b in range(B):
        for r in range(R):
            p = int(mid[b, r])
            for j in range(21):
                x[b, planted[(j + r) % 21], r] = _bump(F, p, 2.0 * 0.8 ** j, g)
        # last row: a very sharp head one column left of the midpoint F - 2.  It loses to the rank-0 head around F - 2,
        # but would win if the midpoint were taken toward F - 1 instead of F (both heads then 0.5 columns away).
        x[b, planted[R % 21], R - 1] = _bump(F, int(mid[b, R - 1]) - 1, 6.0, g)
    qk[:, :, S:S + R, :F] = x
    return qk, jumps.astype(np.int32), B, M, S, R, F


def _dyn_ref(W, count, width, jumps, F):
    """timing.py:94-110 on the softmaxed W [B][LH][R][F] float64 (jumps None: argmax peaks) -> (matrix, kappa)"""
    f = np.arange(F, dtype=np.float64)
    if jumps is None:
        top2 = np.sort(W, -1)[..., -2:]
        m = float(((top2[..., 1] - top2[..., 0]) / top2[..., 1]).min())
        assert m >= 1e-4, f"argmax peaks not separated: {m:.1e}"
        peak = W.argmax(-1).astype(np.float64)[..., None]    # [B][LH][R][1]
    else:
        j1 = np.concatenate([jumps[:, 1:], np.full((jumps.shape[0], 1), F)], 1)
        peak = (jumps + (j1 - jumps) * 0.5)[:, None, :, None]
    scores = (np.abs(peak - f) / 1500 * W).sum(-1)            # [B][LH][R]
    sc = np.swapaxes(scores, 1, 2)                            # [B][R][LH]
    m = _margin(sc, count)
    assert m >= 1e-4, f"head scores not separated at ranks 1..{count + 1}: {m:.1e}"
    heads = np.argsort(sc, -1, kind="stable")[..., :count]    # [B][R][count], slot a = the a-th lowest score
    B, R = heads.shape[:2]
    Wsel = W[np.arange(B)[:, None, None], heads, np.arange(R)[None, :, None]]   # [B][R][count][F]
    ref, kap, _ = _znorm_median_mean(np.swapaxes(Wsel, 1, 2), width)
    return ref, kap


def _dyn_call(L, qk, B, LH, M, S, R, F, scale, width, count, jumps, reuse, ws=None):
    lib = L.lib()
    ldm = (F + 3) // 4 * 4 + 4
    out = torch.full((B, R, ldm), SENTINEL, device="cuda")
    if ws is None:
        ws = torch.zeros(lib.stb_qkpost_dynamic_ws_bytes(B, LH, R, F, count), dtype=torch.uint8, device="cuda")
    L.check(lib.stb_qk_postprocess_dynamic(L.ptr(qk), B, LH, M, LDQ, S, R, F, scale, width, count, L.ptr(jumps), int(reuse),
                                           L.ptr(out), ldm, L.ptr(ws), ws.numel(), L.stream_ptr()))
    torch.cuda.synchronize()
    out = out.cpu()
    assert torch.equal(_bits(out[..., F:]), _bits(torch.full_like(out[..., F:], SENTINEL))), "an output pad column was written"
    return out[..., :F], ws


@pytest.mark.parametrize("count", [1, 6, 20])
@pytest.mark.parametrize("LH", [24, 144, 640, 1280])
def test_dynamic_heads_match_float64(L, LH, count):
    """First iteration (argmax peaks), then prev_jumps with reuse_softmax = 1 on the same workspace; the second result is
    bitwise a fresh call without reuse, and item 1 alone is bitwise item 1 of the batch."""
    qk, jumps, B, M, S, R, F = _dyn_inputs(LH)
    scale, width = {1: (1.0, 7), 6: (0.7, 7), 20: (1.9, 1)}[count]
    sc = float(np.float32(scale))
    W = _softmax(qk[:, :, S:S + R, :F].astype(np.float64) * sc)
    qkd, jd = _dev(qk), _dev(jumps)
    out1, ws = _dyn_call(L, qkd, B, LH, M, S, R, F, scale, width, count, None, 0)
    ref1, kap1 = _dyn_ref(W, count, width, None, F)
    _gate(f"dynamic LH={LH} count={count} first iteration", out1.numpy(), ref1, kap1[:, None, :], DYN_A, DYN_B)
    out2, _ = _dyn_call(L, qkd, B, LH, M, S, R, F, scale, width, count, jd, 1, ws)
    ref2, kap2 = _dyn_ref(W, count, width, jumps, F)
    _gate(f"dynamic LH={LH} count={count} prev_jumps", out2.numpy(), ref2, kap2[:, None, :], DYN_A, DYN_B)
    fresh, _ = _dyn_call(L, qkd, B, LH, M, S, R, F, scale, width, count, jd, 0)
    assert torch.equal(_bits(fresh), _bits(out2)), "reuse_softmax changes the result"
    if B > 1:
        one, _ = _dyn_call(L, qkd[1:2].contiguous(), 1, LH, M, S, R, F, scale, width, count, jd[1:2].contiguous(), 0)
        assert torch.equal(_bits(one[0]), _bits(out2[1])), "item 1 alone differs from item 1 of the batch"


@functools.lru_cache(maxsize=1)
def _new_inputs(LH):
    """qk fp32 [B][LH][M][LDQ] for the new aligner.  21 planted "diagonal" heads (row m peaks at column c0 + 3 m, slope
    1.5 * 0.75^j for rank j) and 3 planted "column" heads (every row peaks at one column, slopes 1.4 / 1.0 / 0.7) that
    rank among the best by column and row norm but lose to the coverage penalty; the other heads are diffuse.  Columns
    >= F are +3e4."""
    B, M, F = {24: (3, 30, 1500), 144: (3, 25, 937), 640: (2, 22, 1500), 1280: (1, 22, 1504)}[LH]
    g = np.random.default_rng(LH + 7)
    qk = np.full((B, LH, M, LDQ), POISON, np.float32)
    x = 0.5 * g.standard_normal((B, LH, M, F), dtype=np.float32)
    planted = _planted(LH, 24, LH + 3)
    c0 = F // 2 - 3 * M // 2
    for j, h in enumerate(planted[:21]):
        for m in range(M):
            x[:, h, m] = _bump(F, c0 + 3 * m, 1.5 * 0.75 ** j, g)
    for k, h in zip((1.4, 1.0, 0.7), planted[21:]):
        c = int(g.integers(20, F - 20))
        for m in range(M):
            x[:, h, m] = _bump(F, c, k, g)
    qk[..., :F] = x
    return qk, B, M, F


def _new_ref(qk, F, scale, width, topk, wc, wr, wv, S, R):
    """timing.py:136-163 in float64, heads in chunks -> (matrix [B][R][F], top-k margin, top-k set with w_coverage = 0)"""
    B, LH, M = qk.shape[:3]
    W = np.empty((B, LH, M, F))
    for h in range(0, LH, 64):
        W[:, h:h + 64] = _softmax(_median(qk[:, h:h + 64, :, :F].astype(np.float64), width) * scale)
    col = np.sqrt((W ** 2).sum(-2))                           # [B][LH][F]
    base = np.zeros((B, LH))
    if wc > 0:
        base += wc * col.sum(-1)
    if wr > 0:
        base += wr * np.sqrt((W ** 2).sum(-1)).sum(-1)
    score = base.copy()
    if wv > 0:
        cov = W.sum(-2)
        score -= wv * (np.maximum(cov, 0.5).sum(-1) - F * 0.5)
    top = np.argsort(-score, -1, kind="stable")[:, :topk]
    s = -np.sort(-score, -1)[:, :topk + 1]
    margin = float(((s[:, :-1] - s[:, 1:]) / np.abs(s[:, :-1])).min())
    top0 = np.argsort(-base, -1, kind="stable")[:, :topk]
    bi = np.arange(B)[:, None]
    ref = (W[bi, top] / col[bi, top][:, :, None, :]).mean(1)[:, S:S + R]
    return ref, margin, top, top0


NEW = [  # LH, topk, (w_colnorm, w_rownorm, w_coverage), qk_scale, medfilt_width
    (24, 1, (1.0, 1.0, 0.0), 1.0, 7),
    (24, 20, (1.0, 1.0, 0.5), 1.3, 7),
    (144, 1, (1.0, 0.0, 0.0), 0.8, 7),
    (144, 20, (0.0, 1.0, 0.0), 1.0, 1),
    (640, 1, (0.0, 1.0, 0.0), 1.0, 7),
    (640, 20, (1.0, 1.0, 0.0), 0.8, 7),
    (1280, 1, (1.0, 1.0, 0.5), 1.0, 7),
    (1280, 20, (1.0, 1.0, 0.5), 1.0, 7),
    (1280, 20, (0.0, 1.0, 0.0), 0.7, 1),
]


@pytest.mark.parametrize("LH,topk,w,scale,width", NEW)
def test_new_aligner_matches_float64(L, LH, topk, w, scale, width):
    """median on the raw scores of all M rows -> softmax -> head score -> top-k -> column-normalised mean, rows
    [S, S+R), against float64 per element; item 1 alone is bitwise item 1 of the batch."""
    qk, B, M, F = _new_inputs(LH)
    S, R = 3, M - 4
    sc = float(np.float32(scale))
    ref, margin, top, top0 = _new_ref(qk, F, sc, width, topk, *w, S, R)
    assert margin >= 1e-4, f"head scores not separated at the top-k cut: {margin:.1e}"
    if w[2] > 0 and topk == 20:
        assert any(set(a) != set(b) for a, b in zip(top, top0)), "the coverage penalty does not change the top-k set"
    lib = L.lib()
    ldm = (F + 3) // 4 * 4 + 4
    qkd = _dev(qk)

    def run(q, nb):
        out = torch.full((nb, R, ldm), SENTINEL, device="cuda")
        ws = torch.zeros(lib.stb_qkpost_new_ws_bytes(nb, LH, M, F, topk), dtype=torch.uint8, device="cuda")
        L.check(lib.stb_qk_postprocess_new(L.ptr(q), nb, LH, M, LDQ, S, R, F, scale, width, topk, *w, L.ptr(out), ldm, L.ptr(ws),
                                           ws.numel(), L.stream_ptr()))
        torch.cuda.synchronize()
        out = out.cpu()
        assert torch.equal(_bits(out[..., F:]), _bits(torch.full_like(out[..., F:], SENTINEL))), "a pad column was written"
        return out[..., :F]

    out = run(qkd, B)
    if B > 1:
        assert torch.equal(_bits(run(qkd[1:2].contiguous(), 1)[0]), _bits(out[1])), "item 1 alone differs"
    o = out.double().numpy()
    assert np.isfinite(o).all() and np.isfinite(ref).all()
    err = float((np.abs(o - ref) / np.abs(ref)).max())
    print(f"new aligner LH={LH} topk={topk} w={w} scale={scale} width={width}: worst |err| / |ref| {err:.2e}, "
          f"top-k margin {margin:.1e}")
    assert err < NEW_BOUND, err


# ---------------------------------------------------------------------------------------------------------------
# token probabilities
# ---------------------------------------------------------------------------------------------------------------
NC, LDL = 50257, 51872


def _logit_rows():
    """fp32 logits [12][LDL] (columns >= NC are filled by the caller) and their targets"""
    g = np.random.default_rng(50257)
    x = (3 * g.standard_normal((12, NC))).astype(np.float32)
    x[4:7] = np.round(x[4:7] * 0.7)                           # quantized: many ties, at the target and at the maximum
    x[7] = 1.75                                               # all equal
    x[8] *= 10                                                # peaky
    x[9] -= 1e4                                               # far from zero
    t = g.integers(0, NC, 12)
    t[0], t[1], t[2], t[6] = 0, NC - 1, x[2].argmax(), 0
    t[5], t[9] = x[5].argmax(), x[9].argmax()
    x[3, t[3]] = -1e4                                         # the target's probability underflows
    x[10, t[10]] = x[10].max() + 0.5                          # a clear maximum on the target
    return x, t.astype(np.int32)


def _token_call(L, x, fill, t):
    buf = np.full((x.shape[0], LDL), fill, np.float32)
    buf[:, :NC] = x
    n = x.shape[0]
    logits, tgt = _dev(buf), _dev(t)                          # held: a freed block could be handed to the next allocation
    prob = torch.full((n,), NAN, device="cuda")
    rank = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    L.check(L.lib().stb_token_probs(L.ptr(logits), LDL, n, NC, L.ptr(tgt), L.ptr(prob), L.ptr(rank), L.stream_ptr()))
    torch.cuda.synchronize()
    return prob.cpu(), rank.cpu()


def test_token_probs_match_float64(L):
    """p = softmax(logits[:n_classes])[target] against float64; the rank bitwise the host count of smaller logits;
    all-equal rows give bitwise fp32(1 / n); columns >= n_classes are NaN, then +1e4, with the same result; a row alone is
    bitwise the row in the batch."""
    x, t = _logit_rows()
    prob, rank = _token_call(L, x, NAN, t)
    p2, r2 = _token_call(L, x, 1e4, t)
    assert torch.equal(_bits(prob), _bits(p2)) and torch.equal(rank, r2), "a logit column >= n_classes was read"
    p5, r5 = _token_call(L, x[5:6], NAN, t[5:6])
    assert torch.equal(_bits(p5), _bits(prob[5:6])) and torch.equal(r5, rank[5:6])
    ref = _softmax(x.astype(np.float64))[np.arange(len(t)), t]
    host_rank = (x < x[np.arange(len(t)), t][:, None]).sum(-1)
    assert np.array_equal(rank.numpy(), host_rank), (rank.numpy(), host_rank)
    assert _bits(prob[7:8]).item() == _bits(torch.tensor([1.0 / NC], dtype=torch.float32)).item(), prob[7].item()
    err = np.abs(prob.double().numpy() - ref) / np.maximum(ref, 2.0 ** -126)
    print(f"token probs: worst |err| / max(p, 2^-126) {err.max():.2e} (p of the -1e4 target {prob[3].item():.1e})")
    assert err.max() < PROB_BOUND, err


def test_softmax_probs_match_float64(L):
    """full probability rows against float64, per row relative to its largest probability; pad columns of the output
    pitch keep a sentinel; all-equal rows are bitwise fp32(1 / n); columns >= n_classes of the logits are NaN."""
    x, _ = _logit_rows()
    n, ldo = x.shape[0], NC + 7
    buf = np.full((n, LDL), np.nan, np.float32)
    buf[:, :NC] = x
    logits = _dev(buf)
    out = torch.full((n, ldo), SENTINEL, device="cuda")
    L.check(L.lib().stb_softmax_probs(L.ptr(logits), LDL, n, NC, L.ptr(out), ldo, L.stream_ptr()))
    torch.cuda.synchronize()
    out = out.cpu()
    assert torch.equal(_bits(out[:, NC:]), _bits(torch.full((n, 7), SENTINEL))), "an output pad column was written"
    p = out[:, :NC]
    assert torch.equal(_bits(p[7]), _bits(torch.full((NC,), 1.0 / NC, dtype=torch.float32)))
    ref = _softmax(x.astype(np.float64))
    err = np.abs(p.double().numpy() - ref).max(-1) / ref.max(-1)
    print(f"softmax probs: worst per-row |err| / max p {err.max():.2e}")
    assert err.max() < SOFTMAX_BOUND, err


# ---------------------------------------------------------------------------------------------------------------
# log-mel
# ---------------------------------------------------------------------------------------------------------------
SIGNALS = ("speech", "quiet speech", "tone on a bin", "tone between bins", "clipped square", "DC + noise", "1e-5 noise",
           "impulse at 0", "impulse at n-1", "zero")


def _signals(n):
    """fp32 [10][n], one row per SIGNALS"""
    from oracle import stable_path as SP
    g = np.random.default_rng(n)
    t = np.arange(n) / 16000.0
    x = np.zeros((len(SIGNALS), n))
    x[0] = SP.synth_audio(n, seed=n % 997).double().numpy()
    x[1] = 0.05 * SP.synth_audio(n, seed=n % 991 + 1).double().numpy()
    x[2] = 0.5 * np.sin(2 * np.pi * 1000.0 * t)              # 1000 Hz: the centre of bin 25 (40 Hz bins)
    x[3] = 0.5 * np.sin(2 * np.pi * 1020.0 * t + 0.3)        # between bins 25 and 26
    x[4] = np.clip(4 * np.sin(2 * np.pi * 440.0 * t), -1, 1)
    x[5] = 0.2 + 0.01 * g.standard_normal(n)
    x[6] = 1e-5 * g.standard_normal(n)
    x[7, 0] = 0.5
    x[8, n - 1] = 0.5
    return x.astype(np.float32)


def _logmel_ref(audio, padded, filters, batch_global):
    """whisper.audio.log_mel_spectrogram in float64 (+ pad_or_trim to 3000 frames) -> (mel [B][n_mels][3000], kappa)"""
    B, n = audio.shape
    x = np.zeros((B, padded))
    x[:, :n] = audio
    xp = np.pad(x, ((0, 0), (200, 200)), mode="reflect")
    nf = min(padded // 160, 3000)                            # 1 + padded // 160 frames, the last one dropped
    k = np.arange(400)
    win = 0.5 - 0.5 * np.cos(2 * np.pi * k / 400)            # periodic Hann
    fr = sliding_window_view(xp, 400, axis=-1)[:, :nf * 160:160] * win
    power = np.abs(np.fft.rfft(fr, axis=-1)) ** 2            # [B][nf][201]
    fil = filters.astype(np.float64)
    P = np.einsum("mk,bfk->bmf", fil, power)
    lg = np.log10(np.maximum(P, 1e-10))
    mx = lg.max() if batch_global else lg.max((1, 2), keepdims=True)
    out = np.zeros((B, fil.shape[0], 3000))
    out[..., :nf] = (np.maximum(lg, mx - 8.0) + 4.0) / 4.0
    E = (fr ** 2).sum(-1)                                    # [B][nf]
    with np.errstate(invalid="ignore", divide="ignore"):
        kap = np.sqrt(E[:, None, :] * fil.sum(-1)[None, :, None] / P)
    kap = np.where(P > 0, kap, 0.0)                          # an all-zero frame: exact
    at_max = lg == mx                                        # a floored element carries the error of the maximum
    kmax = np.where(at_max, kap, 0).max() if batch_global else np.where(at_max, kap, 0).max((1, 2), keepdims=True)
    kap = np.where(lg < mx - 8.0, np.broadcast_to(kmax, kap.shape), kap)
    kp = np.zeros_like(out)
    kp[..., :nf] = kap
    return out, kp


@functools.lru_cache(maxsize=2)
def _mel_model(n_mels):
    """a small random-init model: only its log-mel tables (window, DFT, filterbank) are used"""
    import oracle.whisper_ref as W
    from oracle.whisper_ref.model import ModelDimensions
    from stable_ts_b200.model import from_oracle
    return from_oracle(W.build_model(ModelDimensions(n_mels, 1500, 384, 6, 1, 51864, 448, 384, 6, 1), seed=n_mels))


def _logmel_call(L, audio, padded, n_mels, batch_global, ws_fill):
    """stb_logmel with tables built here, on audio followed by NaN in a longer buffer, into a NaN-filled output"""
    from stable_ts_b200.model import mel_filterbank
    B, n = audio.shape
    k = np.arange(400, dtype=np.float64)
    window = _dev((0.5 - 0.5 * np.cos(2 * np.pi * k / 400)).astype(np.float32))
    dft = _dev(np.stack([np.cos(2 * np.pi * k / 400), np.sin(2 * np.pi * k / 400)], 1).astype(np.float32))
    buf = torch.full((B * n + 4096,), NAN, device="cuda")
    buf[:B * n] = _dev(audio.reshape(-1))
    mel = torch.full((B, n_mels, 3000), NAN, device="cuda")
    filters = _dev(mel_filterbank(n_mels))
    ws = torch.full((B * 376,), ws_fill, device="cuda")
    L.check(L.lib().stb_logmel(L.ptr(buf), B, n, padded, n_mels, L.ptr(filters), L.ptr(window), L.ptr(dft),
                               int(batch_global), L.ptr(mel), L.ptr(ws), ws.numel() * 4, L.stream_ptr()))
    torch.cuda.synchronize()
    return mel.cpu()


LOGMEL = [(n, False) for n in (1, 201, 401, 123457, 479999, 480000)] + \
         [(n, True) for n in (201, 400, 1280, 160 * 13 + 7, 200001, 480000)]


@pytest.mark.parametrize("n_mels", [80, 128])
@pytest.mark.parametrize("n,refine", LOGMEL)
def test_logmel_matches_float64(L, n, refine, n_mels):
    """Ten signals of n samples: align mode pads to 480000 with a per-window maximum, refine mode pads to n with the
    maximum over the batch.  stb_logmel (tables built here) and model.log_mel (the library's tables) against float64; an
    all-zero window is exactly -1.5; refine frames >= n / 160 are exactly 0; the NaN after the audio is never read; a
    NaN-filled workspace gives the same output; each window alone gives its row of the batch."""
    from stable_ts_b200.model import mel_filterbank
    audio = _signals(n)
    padded = n if refine else 480000
    ref, kap = _logmel_ref(audio, padded, mel_filterbank(n_mels), refine)
    out = _logmel_call(L, audio, padded, n_mels, refine, NAN)
    assert not out.isnan().any()
    assert torch.equal(_bits(out), _bits(_logmel_call(L, audio, padded, n_mels, refine, 0.0))), "depends on the workspace"
    if not refine:
        for b in (0, 8, 9):
            assert torch.equal(_bits(out[b]), _bits(_logmel_call(L, audio[b:b + 1], padded, n_mels, False, 0.0)[0])), b
        assert (out[9] == -1.5).all(), "an all-zero window is not exactly -1.5"
    else:
        assert (out[..., n // 160:] == 0).all(), "a refine frame >= n / 160 is not exactly 0"
    lib_out = _mel_model(n_mels).log_mel(_dev(audio), padded_samples=None if not refine else padded,
                                         batch_global_max=refine).cpu()
    mode = "refine" if refine else "align"
    _gate(f"logmel {mode} n={n} mels={n_mels}", out.numpy(), ref, kap, MEL_A, MEL_B)
    _gate(f"model.log_mel {mode} n={n} mels={n_mels}", lib_out.numpy(), ref, kap, MEL_A, MEL_B)
