"""GPU tests of the encoder, the cross K / V and the teacher-forced decoder against float64 references computed on the
CPU, with the LayerNorm and softmax row kernels of those passes on their own (csrc/elementwise.cu, csrc/engine.cu).

- stb_layernorm: every width 128..1280, row counts around the 8-rows-per-CTA grid, rows far from zero mean, constant
  rows, each output alone and all together, rows past the end left untouched.
- stb_softmax_rows: the decoder's causal self-attention rows (slices of M rows at pitch Mp = M rounded up to 8) and the
  cross-attention rows (1500 keys at pitch 1504): near one-hot, all-equal and -1e4 rows, maxima on the diagonal, the
  zero pad columns, and no read of a score outside a row's valid columns.
- stb_encoder_forward on distinct windows (one with a silent tail, one short), with the frames where the conv padding
  enters gated on their own; stb_cross_kv (K head-major, V^T with its zero pad keys) in both layouts;
  stb_decoder_forward logits and captured cross-attention scores for all heads and for an explicit head list; the logits
  bitwise the same whatever is captured, and a head list's scores bitwise those of the same heads in the all-heads pass.
- The same passes on model-owned workspaces filled with NaN give bitwise the same outputs: every pad row, pad key and
  pad column is written before it is read.

The float64 oracle is the fp32 oracle model cast to float64, with its LayerNorm and its attention softmax kept in float64
(the fp32 oracle rounds there).  Each pass is fed this library's own input (log-mel, encoder output), so only that pass
is measured.  Errors are relative to max|ref| of the case.  The bounds are 1.25x the worst error measured on an NVIDIA
H100 80GB HBM3 at 700 W, rounded up to two digits; the measured worsts are next to each bound.

Run on an H100:  python -m pytest tests/test_gpu_forward_fp64.py -q -s
"""
import contextlib
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")
T, TP = 1500, 1504                        # encoder positions; their row pitch in the score / probability / V^T planes

# bounds: 1.25x the worst error measured on an NVIDIA H100 80GB HBM3 at 700 W, rounded up to two digits
LN_BOUND = {0: 2.2e-7,    # LayerNorm vs float64 by the rows' mean / std: worst 1.76e-7
            3: 2.8e-7,    # 2.18e-7
            100: 4.6e-6}  # 3.66e-6 (the fp32 row sum rounds at |sum| ~ 100 d)
SOFTMAX_BOUND = 8.7e-7    # softmax vs float64, per row relative to its largest probability: worst 6.92e-7 (1500 keys, +-40)
# per model, d384 | d1280
ENC_BOUND = {"d384": 9.4e-6, "d1280": 1.4e-5}         # encoder output, worst window: 7.45e-6 | 1.07e-5
ENC_EDGE_BOUND = {"d384": 7.5e-6, "d1280": 1.1e-5}    # output frames 0 and 1499 (conv padding): 5.93e-6 | 8.26e-6
CROSS_KV_BOUND = {"d384": 3.2e-6, "d1280": 7.7e-6}    # cross K and V^T on the xa planes they read: 2.50e-6 | 6.13e-6
LOGITS_BOUND = {"d384": 9.4e-6, "d1280": 1.5e-5}      # teacher-forced logits: 7.45e-6 | 1.16e-5
QK_BOUND = {"d384": 9.3e-6, "d1280": 2.2e-5}          # captured cross-attention scores: 7.43e-6 | 1.70e-5

DIMS = {  # (n_mels, n_audio_ctx, n_audio_state, n_audio_head, n_audio_layer, n_vocab, n_text_ctx, n_text_state, n_text_head,
          #  n_text_layer), model seed, windows (samples of synthetic audio, samples kept before silence), encoder batch
    "d384": ((80, 1500, 384, 6, 2, 51864, 448, 384, 6, 2), 23, [(480000, None), (480000, 200000), (100000, None)]),
    "d1280": ((128, 1500, 1280, 20, 1, 51866, 448, 1280, 20, 2), 17, [(480000, None), (150000, None)]),
}
# an explicit head selection per model: unsorted, one pair twice, pairs from the last layer only
HEADS = {"d384": [(1, 4), (1, 0), (1, 4), (1, 5), (1, 2)], "d1280": [(1, 17), (1, 3), (1, 17), (1, 0), (1, 19), (1, 8)]}


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from stable_ts_b200 import _lib
    _lib.lib()
    return _lib


def _bits(t):
    """bit pattern of a float tensor (bitwise comparisons that NaN cannot spoil)"""
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def _split(y):
    """fp16 split of fp32 values: hi = rn(y), lo = rn(y - hi)"""
    hi = y.half()
    return hi, (y - hi.float()).half()


def _rel(out, ref):
    return ((out.double().cpu() - ref).abs().max() / ref.abs().max()).item()


@contextlib.contextmanager
def _float64_oracle():
    """The oracle's LayerNorm casts to fp32 and its attention rounds the scores to fp32 before the softmax; keep both in
    float64, and always return the scaled pre-softmax scores (what the cross-attention capture writes)."""
    import torch.nn.functional as F
    from oracle.whisper_ref import model as WM

    def qkv_attention(self, q, k, v, mask=None):
        n_ctx, n_state = q.shape[1], q.shape[2]
        scale = (n_state // self.n_head) ** -0.25
        q = q.view(*q.shape[:2], self.n_head, -1).permute(0, 2, 1, 3)
        k = k.view(*k.shape[:2], self.n_head, -1).permute(0, 2, 1, 3)
        v = v.view(*v.shape[:2], self.n_head, -1).permute(0, 2, 1, 3)
        qk = (q * scale) @ (k * scale).transpose(-1, -2)
        if mask is not None:
            qk = qk + mask[:n_ctx, :n_ctx]
        out = (F.softmax(qk, dim=-1) @ v).permute(0, 2, 1, 3).flatten(start_dim=2)
        return out, qk

    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        mp.setattr(WM.LayerNorm, "forward", lambda self, x: F.layer_norm(x, self.normalized_shape, self.weight, self.bias, self.eps))
        mp.setattr(WM.MultiHeadAttention, "qkv_attention", qkv_attention)
        yield


class Case:
    """A random-init model on the device and in float64 on the CPU, its windows' log-mel (this library's) and encoder
    output; the float64 encoder output is computed on first use."""

    def __init__(self, name):
        import oracle.whisper_ref as W
        from oracle import stable_path as SP
        from oracle.whisper_ref.model import ModelDimensions
        from stable_ts_b200.model import from_oracle
        dims, seed, windows = DIMS[name]
        self.model = W.build_model(ModelDimensions(*dims), seed=seed)
        self.m64 = copy.deepcopy(self.model).double()
        self.gm = from_oracle(self.model)
        audio = torch.zeros(len(windows), 480000)
        for b, (n, keep) in enumerate(windows):
            audio[b, :n] = SP.synth_audio(n, seed=100 * seed + b)
            if keep is not None:
                audio[b, keep:] = 0                           # a silent tail
        self.mel = self.gm.log_mel(audio.cuda())
        self.enc = self.gm.encode(self.mel)
        torch.cuda.synchronize()
        self.B = len(windows)
        self._xa_ref = None

    def xa_ref(self):
        if self._xa_ref is None:
            mel = self.mel.double().cpu()
            with _float64_oracle():
                self._xa_ref = torch.cat([self.m64.encoder(mel[b:b + 1]) for b in range(self.B)])
        return self._xa_ref


@pytest.fixture(scope="module")
def cases(L):
    made = {}

    def get(name):
        if name not in made:
            made[name] = Case(name)
        return made[name]

    yield get
    made.clear()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# LayerNorm on its own
# ---------------------------------------------------------------------------------------------------------------
def _ln_rows(rows, d, g):
    """rows of N(0, 1) shifted by a mean of 0, 3 or 100 (mean / std), every fourth row constant; -> x fp32, kind per row
    (-1: constant)"""
    kind = torch.tensor([0, 3, 100, -1]).repeat(rows // 4 + 1)[:rows]
    x = torch.randn(rows, d, generator=g, dtype=torch.float64) + kind.clamp(min=0)[:, None]
    x[kind < 0] = -1.25                                       # exact in fp32: the row's fp32 mean is exact, its variance 0
    return x.float(), kind


def _ln_ref(x, gamma, beta):
    x = x.double()
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return (x - mean) / (var + 1e-5).sqrt() * gamma.double().cpu() + beta.double().cpu()


def _ln_call(L, x, d, gamma, beta, planes):
    """LayerNorm of x [rows][d] into outputs of rows + 9 rows filled with NaN; checks that the rows past `rows` are left
    untouched and returns (f32, hi, lo) of the first `rows` rows (None where not asked for)"""
    rows = x.shape[0]
    f32 = torch.full((rows + 9, d), NAN, device="cuda") if "f32" in planes else None
    hi = torch.full((rows + 9, d), NAN, dtype=torch.float16, device="cuda") if "hi" in planes else None
    lo = torch.full((rows + 9, d), NAN, dtype=torch.float16, device="cuda") if "lo" in planes else None
    L.check(L.lib().stb_layernorm(L.ptr(x), rows, d, L.ptr(gamma), L.ptr(beta), L.ptr(hi), L.ptr(lo), L.ptr(f32),
                                  L.stream_ptr()))
    torch.cuda.synchronize()
    out = []
    for t, fill in ((f32, torch.full((9, d), NAN)), (hi, torch.full((9, d), NAN).half()), (lo, torch.full((9, d), NAN).half())):
        if t is not None:
            assert torch.equal(_bits(t[rows:].cpu()), _bits(fill)), "a row past the end was written"
        out.append(None if t is None else t[:rows].cpu())
    return out


@pytest.mark.parametrize("d", list(range(128, 1281, 128)))
def test_layernorm_matches_float64(L, d):
    """Every width (d / 128 float4 per lane), 1 / 7 / 8 / 9 / 4501 rows; the fp32 output against float64 by mean / std;
    constant rows give beta exactly; the planes are the split of the fp32 output; each output alone is bitwise the same."""
    g = torch.Generator().manual_seed(d)
    gamma = (1 + 0.5 * (2 * torch.rand(d, generator=g) - 1)).cuda()
    beta = (0.5 * torch.randn(d, generator=g)).cuda()
    worst = {k: 0.0 for k in LN_BOUND}
    for rows in (1, 7, 8, 9, 4501):
        x, kind = _ln_rows(rows, d, g)
        xd = x.cuda()
        f32, hi, lo = _ln_call(L, xd, d, gamma, beta, "f32 hi lo")
        ref = _ln_ref(x, gamma, beta)
        for k in LN_BOUND:
            sel = kind == k
            if sel.any():
                worst[k] = max(worst[k], _rel(f32[sel], ref[sel]))
        if (kind < 0).any():                                  # variance 0: (x - mean) rstd is exactly 0
            assert torch.equal(f32[kind < 0], beta.cpu().expand(int((kind < 0).sum()), d))
        h, l = _split(f32)
        assert torch.equal(_bits(hi), _bits(h)) and torch.equal(_bits(lo), _bits(l))
        assert torch.equal(_bits(_ln_call(L, xd, d, gamma, beta, "f32")[0]), _bits(f32))
        assert torch.equal(_bits(_ln_call(L, xd, d, gamma, beta, "hi")[1]), _bits(hi))
        _, hi2, lo2 = _ln_call(L, xd, d, gamma, beta, "hi lo")
        assert torch.equal(_bits(hi2), _bits(hi)) and torch.equal(_bits(lo2), _bits(lo))
    print(f"layernorm d={d}: worst rel err by mean/std " + ", ".join(f"{k}: {v:.2e}" for k, v in worst.items()))
    for k, v in worst.items():
        assert v < LN_BOUND[k], (k, v)


# ---------------------------------------------------------------------------------------------------------------
# softmax rows on their own
# ---------------------------------------------------------------------------------------------------------------
SM_KINDS = ("std 3", "spread +-40", "all equal", "around -1e4", "std 3, max last", "spread +-40, max last")


def _scores(valid, ld, kind, g):
    """S fp32 [rows][ld]: row r of kind kind[r] (SM_KINDS) over its valid[r] columns, NaN elsewhere ("max last": the
    row's largest score sits on its last valid column, the diagonal of a causal slice)"""
    rows = len(valid)
    gen = torch.stack([3 * torch.randn(rows, ld, generator=g, dtype=torch.float64),
                       80 * torch.rand(rows, ld, generator=g, dtype=torch.float64) - 40,
                       torch.full((rows, ld), 1.75, dtype=torch.float64),
                       -1e4 + 3 * torch.randn(rows, ld, generator=g, dtype=torch.float64)])
    S = gen[kind % 4, torch.arange(rows)].float()
    col = torch.arange(ld)[None, :]
    inside = col < valid[:, None]
    last = kind >= 4
    mx = torch.where(inside, S, torch.tensor(-float("inf"))).amax(1)
    S[last, valid[last] - 1] = mx[last] + 2
    return torch.where(inside, S, torch.tensor(NAN))         # NaN: a score the kernel must not read


def _softmax_check(L, S, valid, kind, n_cols, ld, causal, rows_per_slice):
    """run stb_softmax_rows on S (with and without the lo plane) into NaN-filled planes with a NaN guard after them;
    all-equal rows must be exactly the split of fp32(1 / n).  Returns, for the other kinds, the worst per-row error vs
    float64 relative to the row's largest probability (hi + lo carries an absolute error of up to 2^-25 where lo is
    subnormal, so rows whose largest probability is small are not a fair test of the kernel's fp32 arithmetic)"""
    n_rows = S.shape[0]
    planes = []
    for with_lo in (True, False):
        hi = torch.full((n_rows * ld + 64,), NAN, dtype=torch.float16, device="cuda")
        lo = torch.full_like(hi, NAN) if with_lo else None
        L.check(L.lib().stb_softmax_rows(L.ptr(S.cuda()), n_rows, n_cols, ld, rows_per_slice, int(causal), L.ptr(hi), L.ptr(lo),
                                         ld, L.stream_ptr()))
        torch.cuda.synchronize()
        planes.append((hi.cpu(), None if lo is None else lo.cpu()))
    (hi, lo), (hi1, _) = planes
    assert torch.equal(_bits(hi1), _bits(hi)), "the hi plane depends on whether lo is written"
    guard = torch.full((64,), NAN).half()
    assert torch.equal(_bits(hi[n_rows * ld:]), _bits(guard)) and torch.equal(_bits(lo[n_rows * ld:]), _bits(guard))
    hi, lo = hi[:n_rows * ld].view(n_rows, ld), lo[:n_rows * ld].view(n_rows, ld)
    pad = torch.arange(ld)[None, :] >= valid[:, None]
    assert (_bits(hi)[pad] == 0).all() and (_bits(lo)[pad] == 0).all(), "a pad column is not +0"
    p = hi.double() + lo.double()
    ref = torch.where(pad, torch.tensor(-float("inf"), dtype=torch.float64), S.double().nan_to_num(0.0)).softmax(-1)
    err = ((p - ref).abs().amax(1) / ref.amax(1))
    eq = kind == 2                                            # all-equal rows: exactly the split of fp32(1 / n)
    inv = (1.0 / valid[eq].double()).float()
    h, l = _split(inv[:, None].expand(-1, ld).contiguous())
    assert torch.equal(_bits(hi[eq])[~pad[eq]], _bits(h)[~pad[eq]]) and torch.equal(_bits(lo[eq])[~pad[eq]], _bits(l)[~pad[eq]])
    return {k: err[kind == i].max().item() for i, k in enumerate(SM_KINDS) if i != 2 and (kind == i).any()}


@pytest.mark.parametrize("M", [1, 7, 8, 9, 64, 65, 447, 448])
def test_causal_softmax_matches_float64(L, M):
    """The decoder's self-attention rows: B = 3, H = 6 slices of M rows at pitch Mp (M rounded up to 8); row r of a slice
    covers columns 0..r.  Each kind of row fills three slices."""
    Mp = (M + 7) // 8 * 8
    g = torch.Generator().manual_seed(M)
    n_rows = 18 * M
    r = torch.arange(n_rows)
    valid = r % M + 1
    kind = (r // M) % len(SM_KINDS)
    S = _scores(valid, Mp, kind, g)
    worst = _softmax_check(L, S, valid, kind, M, Mp, True, M)
    print(f"causal softmax M={M}: worst rel err " + ", ".join(f"{k}: {v:.2e}" for k, v in worst.items()))
    assert max(worst.values()) < SOFTMAX_BOUND, worst


def test_cross_softmax_matches_float64(L):
    """The cross-attention rows: 1500 keys at pitch 1504, 51 rows (a partial 8-row CTA), every kind of row; columns
    1500..1503 are exactly 0."""
    g = torch.Generator().manual_seed(1500)
    n_rows = 51
    valid = torch.full((n_rows,), T)
    kind = torch.arange(n_rows) % len(SM_KINDS)
    S = _scores(valid, TP, kind, g)
    worst = _softmax_check(L, S, valid, kind, T, TP, False, 1)
    print("cross softmax 1500 / 1504: worst rel err " + ", ".join(f"{k}: {v:.2e}" for k, v in worst.items()))
    assert max(worst.values()) < SOFTMAX_BOUND, worst


# ---------------------------------------------------------------------------------------------------------------
# encoder, cross K / V, teacher-forced decoder
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["d384", "d1280"])
def test_encoder_matches_float64(cases, name):
    """Encoder output of distinct windows (d384: B = 3 with a silent tail and a short window; d1280: B = 2, 128 mels)
    against the float64 encoder on the same log-mel; output frames 0 and 1499 on their own; the xa planes are the split
    of the fp32 output."""
    c = cases(name)
    xa = c.enc["f32"].double().cpu()
    ref = c.xa_ref()
    worst = worst_edge = 0.0
    for b in range(c.B):
        den = ref[b].abs().max()
        e = ((xa[b] - ref[b]).abs().max() / den).item()
        e_edge = max(((xa[b, t] - ref[b, t]).abs().max() / den).item() for t in (0, T - 1))
        print(f"encoder {name} window {b}: rel err {e:.2e}, frames 0 / 1499 {e_edge:.2e}")
        worst, worst_edge = max(worst, e), max(worst_edge, e_edge)
    assert worst < ENC_BOUND[name] and worst_edge < ENC_EDGE_BOUND[name], (worst, worst_edge)
    h, l = _split(c.enc["f32"].view(c.B * T, -1))
    assert torch.equal(_bits(c.enc["hi"]), _bits(h)) and torch.equal(_bits(c.enc["lo"]), _bits(l))


def _cross_kv_planes(gm, blk, B, l):
    """(K hi, K lo [B][H][T][64], V^T hi, V^T lo [B][H][64][1504]) of decoder layer l in a stb_cross_kv block"""
    D = gm.dims
    d, H = D.n_text_state, D.n_text_head
    k_el, v_el = B * T * d, B * d * TP
    per = 2 * (2 * k_el + v_el) + k_el
    p = blk.view(torch.float16)[l * per:(l + 1) * per]
    return (p[:k_el].view(B, H, T, 64), p[k_el:2 * k_el].view(B, H, T, 64), p[2 * k_el:2 * k_el + v_el].view(B, H, 64, TP),
            p[2 * k_el + v_el:2 * k_el + 2 * v_el].view(B, H, 64, TP))


@pytest.mark.parametrize("name", ["d384", "d1280"])
def test_cross_kv_matches_float64(L, cases, name):
    """K head-major and V^T (with the V bias) of every decoder layer against float64 on the xa planes they read (hi + lo);
    V^T keys 1500..1503 exactly 0; both layouts give bitwise the same K and V^T."""
    c = cases(name)
    gm, B = c.gm, c.B
    D = gm.dims
    d, H = D.n_text_state, D.n_text_head
    xa = (c.enc["hi"].double() + c.enc["lo"].double()).cpu().view(B, T, d)
    nbytes = gm._lib.stb_cross_kv_bytes(gm._h, B)
    blocks = []
    for layout in (0, 1):
        blk = torch.full((nbytes // 2,), -1, dtype=torch.int16, device="cuda")       # 0xFFFF: NaN in every fp16
        L.check(gm._lib.stb_cross_kv(gm._h, L.ptr(c.enc["hi"]), L.ptr(c.enc["lo"]), B, layout, L.ptr(blk), L.stream_ptr()))
        torch.cuda.synchronize()
        blocks.append(blk)
    worst = 0.0
    for l in range(D.n_text_layer):
        a = _cross_kv_planes(gm, blocks[0], B, l)
        b = _cross_kv_planes(gm, blocks[1], B, l)
        for x, y in zip(a, b):
            assert torch.equal(_bits(x), _bits(y)), f"layer {l}: the layouts differ"
        ca = c.model.decoder.blocks[l].cross_attn
        with torch.no_grad():
            K = (xa @ ca.key.weight.double().T).view(B, T, H, 64).permute(0, 2, 1, 3)
            V = (xa @ ca.value.weight.double().T + ca.value.bias.double()).view(B, T, H, 64).permute(0, 2, 3, 1)
        k_hi, k_lo, v_hi, v_lo = (t.cpu() for t in a)
        e_k = _rel(k_hi.double() + k_lo.double(), K)
        e_v = _rel(v_hi[..., :T].double() + v_lo[..., :T].double(), V)
        print(f"cross K / V^T {name} layer {l}: rel err K {e_k:.2e}, V^T {e_v:.2e}")
        worst = max(worst, e_k, e_v)
        assert (_bits(v_hi[..., T:]) == 0).all() and (_bits(v_lo[..., T:]) == 0).all(), "a V^T pad key is not +0"
    assert worst < CROSS_KV_BOUND[name], worst


def _decoder_inputs(c, M, seed):
    """three token rows of M different random tokens, and the encoder output the decoder reads (d1280 encodes two
    windows: its third row reads the first window again) as (xa planes dict for stb_cross_kv, fp32 [3][T][d])"""
    g = torch.Generator().manual_seed(seed)
    tokens = torch.randint(0, c.gm.dims.n_vocab, (3, M), generator=g, dtype=torch.int32)
    idx = [b % c.B for b in range(3)]
    d = c.gm.dims.n_audio_state
    pick = lambda t: torch.cat([t.view(c.B, T, d)[i] for i in idx]).contiguous()
    enc = {"hi": pick(c.enc["hi"]), "lo": pick(c.enc["lo"]), "B": 3}
    return tokens, enc, c.enc["f32"][idx]


@pytest.mark.parametrize("name,M", [("d384", 1), ("d384", 9), ("d384", 64), ("d384", 65), ("d384", 448), ("d1280", 1),
                                    ("d1280", 65), ("d1280", 448)])
def test_teacher_forced_decoder_matches_float64(cases, name, M):
    """Every logit of three distinct token rows, and the captured scaled pre-softmax cross-attention scores (columns
    0..1499) of all heads and of an explicit head list, against the float64 decoder on this library's encoder output.
    The logits are bitwise the same with no capture, a head list or all heads; the head list's scores are bitwise those
    of the same heads in the all-heads pass."""
    c = cases(name)
    gm = c.gm
    D = gm.dims
    H = D.n_text_head
    tokens, enc, xa = _decoder_inputs(c, M, seed=1000 + M)
    ckv = gm.cross_kv(enc)
    logits, qk = gm.decode_forced(tokens, ckv, heads="all")
    _, qk_sel = gm.decode_forced(tokens, ckv, want_logits=False, heads=HEADS[name])
    logits_none, _ = gm.decode_forced(tokens, ckv)
    logits_sel, _ = gm.decode_forced(tokens, ckv, heads=HEADS[name])
    torch.cuda.synchronize()
    for what, other in (("no capture", logits_none), ("a head list", logits_sel)):
        assert torch.equal(_bits(other), _bits(logits)), f"the logits with {what} differ from those with all heads captured"
    for i, (l, h) in enumerate(HEADS[name]):
        assert torch.equal(_bits(qk_sel[:, i, :, :T]), _bits(qk[:, l * H + h, :, :T])), f"head list slot {i} ({l}, {h})"
    qks = [None] * D.n_text_layer
    hooks = [blk.cross_attn.register_forward_hook(lambda _m, _i, out, i=i: qks.__setitem__(i, out[-1]))
             for i, blk in enumerate(c.m64.decoder.blocks)]
    try:
        with _float64_oracle():
            ref = c.m64.decoder(tokens.long(), xa.double().cpu())
    finally:
        for h in hooks:
            h.remove()
    e_logits = _rel(logits, ref.double())
    del ref
    e_all = max(_rel(qk[:, l * H:(l + 1) * H, :, :T], qks[l]) for l in range(D.n_text_layer))
    e_sel = max(_rel(qk_sel[:, i, :, :T], qks[l][:, h]) for i, (l, h) in enumerate(HEADS[name]))
    print(f"decoder {name} M={M}: rel err logits {e_logits:.2e}, qk all heads {e_all:.2e}, qk head list {e_sel:.2e}")
    assert e_logits < LOGITS_BOUND[name] and e_all < QK_BOUND[name] and e_sel < QK_BOUND[name], (e_logits, e_all, e_sel)


def test_padding_is_written_before_it_is_read(cases):
    """Encoder, cross K / V and decoder once; then the model-owned workspaces filled with 0xFF (a NaN in every float) and
    the same again: xa, the logits and the captured scores must be bitwise the same.  Covers the conv pad rows, the V^T pad
    keys, the probability pad columns and the Mp padding of the decoder's self-attention."""
    c = cases("d384")
    gm = c.gm
    for M in (9, 65):
        tokens = _decoder_inputs(c, M, seed=2000 + M)[0]

        def run():
            enc = gm.encode(c.mel)
            ckv = gm.cross_kv(enc, reuse=True)
            logits, qk = gm.decode_forced(tokens, ckv, heads="all")
            torch.cuda.synchronize()
            return [enc["f32"].clone(), enc["hi"].clone(), enc["lo"].clone(), logits.clone(), qk[..., :T].clone()]

        first = run()
        for ws in ("enc", "cross_kv", "dec"):
            gm._ws[ws].fill_(255)
        second = run()
        for what, a, b in zip(("xa f32", "xa hi", "xa lo", "logits", "qk"), first, second):
            assert not a.isnan().any(), what
            assert torch.equal(_bits(a), _bits(b)), f"M={M}: {what} depends on the workspace's old contents"
