"""GPU tests of the decode step's two attention kernels against float64 references computed on the CPU:
stb_decode_self_attn (the self-attention over the fp32 K/V cache) and stb_decode_cross_attn (the tensor-core
cross-attention over the window's fp16 K / V), csrc/decode.cu.

Self-attention: positions on both sides of the 16-key lane groups and the 64-key loop, deep caches (2 n_text_ctx rows),
the cache row it writes and the rows it must never read (ragged first rows, an idle right-aligned sequence), a cache
built one step at a time on a device counter, peaked / flat / uniform weights, and the output planes.
Cross-attention: every Whisper head count, the zero-filled keys past 1500, a dominant key at every split edge, the merge
of split partials with different maxima, the tickets and scratch across launches, the output planes, and the head-major
V copy stb_cross_kv writes for it.
Then whole decode steps to the end of the context with ragged prompts, against the oracle's decode in float64, and the
same run on a stale model-owned cache.

Errors are relative to max|ref| of the case.  The bounds are 1.25x the worst error measured on an NVIDIA H100 80GB HBM3
at 700 W, rounded up; the measured worsts are next to each bound.

Run on an H100:  python -m pytest tests/test_gpu_decode_attention.py -q -s
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")
T = 1500                                  # encoder positions: keys of the cross-attention
SCALE = 0.125                             # 1 / sqrt(64)

# bounds: 1.25x the worst error measured on an NVIDIA H100 80GB HBM3 at 700 W, rounded up
SELF_BOUND = 7e-7           # self-attention vs float64, scores with a standard deviation of 3: worst 5.30e-7
SELF_PEAKED_BOUND = 3e-6    # self-attention, near one-hot weights (scores spread +-100): worst 1.77e-6
CROSS_BOUND = 1e-6          # cross-attention vs float64 on the fp16 K / V it reads, every cross test: worst 7.65e-7
STEP_BOUND = 2e-5           # step logits vs the float64 oracle to the end of the context: worst 1.13e-5 (B = 3), 1.19e-5 (B = 21)


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from stable_ts_b200 import _lib
    _lib.lib()
    return _lib


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rel(out, ref):
    return ((out.double().cpu() - ref).abs().max() / ref.abs().max()).item()


def _bits(t):
    """bit pattern of a float tensor (bitwise comparisons that NaN cannot spoil)"""
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


class Out:
    """Output planes [B][d] filled with NaN: f32 and / or the fp16 hi / lo split."""

    def __init__(self, B, d, planes="f32"):
        self.f32 = torch.full((B, d), NAN, device="cuda") if "f32" in planes else None
        self.hi = torch.full((B, d), NAN, dtype=torch.float16, device="cuda") if "hi" in planes else None
        self.lo = torch.full((B, d), NAN, dtype=torch.float16, device="cuda") if "lo" in planes else None

    def value(self):
        """what was computed, as float64 on the CPU"""
        if self.f32 is not None:
            return self.f32.double().cpu()
        v = self.hi.double()
        if self.lo is not None:
            v = v + self.lo.double()
        return v.cpu()


def _check_split(out, o32):
    """hi / lo planes must be the fp16 split of the fp32 output: hi = rn(o), lo = rn(o - hi)"""
    hi = o32.half()
    assert torch.equal(_bits(out.hi), _bits(hi))
    if out.lo is not None:
        assert torch.equal(_bits(out.lo), _bits((o32 - hi.float()).half()))


# ---------------------------------------------------------------------------------------------------------------
# self-attention over the fp32 K/V cache
# ---------------------------------------------------------------------------------------------------------------
def _self_call(L, qkv, Kc, Vc, H, pos, seq_off=None, planes="f32"):
    B, rows = Kc.shape[0], Kc.shape[1]
    out = Out(B, 64 * H, planes)
    L.check(L.lib().stb_decode_self_attn(L.ptr(qkv), L.ptr(Kc), L.ptr(Vc), B, H, rows, L.ptr(pos), L.ptr(seq_off),
                                         L.ptr(out.f32), L.ptr(out.hi), L.ptr(out.lo), L.stream_ptr()))
    torch.cuda.synchronize()
    return out


def _self_ref(qkv, Kc, Vc, H, pos, seq_off=None):
    """float64 softmax(q . K[j] / 8, j in [first_row, pos]) V per (sequence, head), from the caches as the kernel left them"""
    B, d = qkv.shape[0], 64 * H
    q = qkv[:, :d].double().cpu().view(B, H, 64)
    out = torch.empty(B, H, 64, dtype=torch.float64)
    for b in range(B):
        first = 0 if seq_off is None else min(int(seq_off[b]), pos)
        K = Kc[b, first:pos + 1].double().cpu().view(-1, H, 64)
        V = Vc[b, first:pos + 1].double().cpu().view(-1, H, 64)
        p = (torch.einsum("jhc,hc->hj", K, q[b]) * SCALE).softmax(-1)
        out[b] = torch.einsum("hj,jhc->hc", p, V)
    return out.view(B, d)


def _self_inputs(B, H, rows, pos, seed, sigma=3 ** 0.5, fill=NAN):
    """qkv [B][3d] and caches [B][rows][d]: rows < pos random, rows >= pos `fill`.  q and k ~ N(0, sigma^2): scores
    q . k / 8 have a standard deviation of sigma^2; v ~ N(0, 1)"""
    d = 64 * H
    g = _gen(seed)
    qkv = torch.randn(B, 3 * d, device="cuda", generator=g)
    qkv[:, : 2 * d] *= sigma
    Kc = torch.full((B, rows, d), fill, device="cuda")
    Vc = torch.full((B, rows, d), fill, device="cuda")
    Kc[:, :pos] = torch.randn(B, pos, d, device="cuda", generator=g) * sigma
    Vc[:, :pos] = torch.randn(B, pos, d, device="cuda", generator=g)
    return qkv, Kc, Vc


def _pos(p):
    return torch.tensor([p], dtype=torch.int32, device="cuda")


def _expect_written(Kc0, Vc0, qkv, H, pos):
    """the caches as they must be after the call: row pos of every sequence holds the k / v slices of qkv"""
    d = 64 * H
    K, V = Kc0.clone(), Vc0.clone()
    K[:, pos] = qkv[:, d:2 * d]
    V[:, pos] = qkv[:, 2 * d:]
    return K, V


# n = pos + 1 keys: one key, one / all / more than the 16 lane groups, one / two 64-key iterations, a full n_text_ctx cache
# and the last row of a 2 n_text_ctx cache (ragged prompts); H = 6 (tiny) and 20 (large-v3); B = 1, 5, 128
SELF_CASES = [(1, 448, 6, 1), (2, 448, 20, 5), (15, 448, 6, 5), (16, 448, 20, 1), (17, 448, 6, 128), (63, 448, 20, 5),
              (64, 448, 6, 5), (65, 448, 20, 5), (128, 448, 6, 128), (129, 448, 20, 1), (448, 448, 20, 5),
              (448, 448, 6, 128), (896, 896, 20, 5), (896, 896, 6, 1)]


@pytest.mark.parametrize("n,rows,H,B", SELF_CASES)
def test_self_attn_positions_vs_fp64(L, n, rows, H, B):
    pos = n - 1
    sentinel = 12345.5                                     # rows >= pos before the call: must stay bitwise, except row pos
    qkv, Kc, Vc = _self_inputs(B, H, rows, pos, seed=n * 31 + H + B, fill=sentinel)
    K0, V0 = _expect_written(Kc, Vc, qkv, H, pos)
    out = _self_call(L, qkv, Kc, Vc, H, _pos(pos))
    assert torch.equal(_bits(Kc), _bits(K0)) and torch.equal(_bits(Vc), _bits(V0)), "cache rows other than pos changed"
    err = _rel(out.value(), _self_ref(qkv, Kc, Vc, H, pos))
    print(f"self-attn n={n} rows={rows} H={H} B={B}: rel err {err:.3e}")
    assert err < SELF_BOUND


@pytest.mark.parametrize("H,pos", [(6, 200), (20, 447), (6, 895)])
def test_self_attn_ragged_rows_are_never_read(L, H, pos):
    """first rows 0, 1, 63, 64, pos and one idle sequence (seq_off > pos: its one key is row pos); every row below a
    sequence's first row and above pos is NaN"""
    rows = 896 if pos >= 448 else 448
    offs = [0, 1, 63, 64, pos, pos + 37]
    B = len(offs)
    qkv, Kc, Vc = _self_inputs(B, H, rows, pos, seed=pos + H)
    for b, o in enumerate(offs):
        Kc[b, : min(o, pos)] = NAN
        Vc[b, : min(o, pos)] = NAN
    seq_off = torch.tensor(offs, dtype=torch.int32, device="cuda")
    out = _self_call(L, qkv, Kc, Vc, H, _pos(pos), seq_off)
    o = out.value()
    assert torch.isfinite(o).all(), "a NaN row outside [first_row, pos] was read"
    err = _rel(o, _self_ref(qkv, Kc, Vc, H, pos, offs))
    print(f"self-attn ragged H={H} pos={pos} first rows {offs}: rel err {err:.3e}")
    assert err < SELF_BOUND
    d = 64 * H
    for b in (4, 5):                                       # one key: p = l = 1, the merge adds zeros only
        assert torch.equal(out.f32[b], qkv[b, 2 * d:]), f"sequence {b} (seq_off {offs[b]}) != V row pos"


def test_self_attn_cache_built_on_a_device_counter(L):
    """300 calls, pos incremented on the device between them as the decode loop does, ragged first rows; every step against
    float64; at the end the caches hold exactly the k / v rows that were fed"""
    H, B, rows = 6, 5, 300
    d = 64 * H
    offs = [0, 3, 64, 150, 299]
    seq_off = torch.tensor(offs, dtype=torch.int32, device="cuda")
    Kc = torch.full((B, rows, d), NAN, device="cuda")
    Vc = torch.full((B, rows, d), NAN, device="cuda")
    g = _gen(77)
    pos = _pos(0)
    feed = []
    worst = 0.0
    for p in range(rows):
        qkv = torch.randn(B, 3 * d, device="cuda", generator=g)
        qkv[:, : 2 * d] *= 3 ** 0.5
        feed.append(qkv)
        out = _self_call(L, qkv, Kc, Vc, H, pos, seq_off)
        worst = max(worst, _rel(out.value(), _self_ref(qkv, Kc, Vc, H, p, offs)))
        pos += 1                                           # on the device
    print(f"self-attn 300 steps on a device counter: worst rel err {worst:.3e}")
    assert worst < SELF_BOUND
    assert int(pos) == rows
    fed = torch.stack(feed, 1)                             # [B][rows][3d]
    assert torch.equal(_bits(Kc), _bits(fed[:, :, d:2 * d].contiguous()))
    assert torch.equal(_bits(Vc), _bits(fed[:, :, 2 * d:].contiguous()))


@pytest.mark.parametrize("kind", ["one_hot", "equal_keys", "tiny_q"])
def test_self_attn_weight_distributions(L, kind):
    H, B, rows, pos = 20, 5, 448, 199
    sigma = 30 ** 0.5 if kind == "one_hot" else 3 ** 0.5      # score spread ~ +-100 for the near one-hot case
    qkv, Kc, Vc = _self_inputs(B, H, rows, pos, seed=5 + len(kind), sigma=sigma)
    d = 64 * H
    if kind == "equal_keys":                                # every key equal: the mean of V
        Kc[:, :pos] = qkv[:, None, d:2 * d]
    if kind == "tiny_q":                                    # q at 1e-3: uniform weights
        qkv[:, :d] *= 1e-3 / sigma
    out = _self_call(L, qkv, Kc, Vc, H, _pos(pos))
    ref = _self_ref(qkv, Kc, Vc, H, pos)
    err = _rel(out.value(), ref)
    if kind == "equal_keys":
        mean_v = Vc[:, : pos + 1].double().cpu().mean(1)
        assert _rel(ref, mean_v) < 1e-12
        err = max(err, _rel(out.value(), mean_v))
    print(f"self-attn {kind}: rel err {err:.3e}")
    assert err < (SELF_PEAKED_BOUND if kind == "one_hot" else SELF_BOUND)


def test_self_attn_output_planes(L):
    H, B, rows, pos = 20, 5, 448, 130
    qkv, Kc, Vc = _self_inputs(B, H, rows, pos, seed=99)
    f = _self_call(L, qkv, Kc, Vc, H, _pos(pos), planes="f32")
    err = _rel(f.value(), _self_ref(qkv, Kc, Vc, H, pos))
    for planes in ("hi+lo", "hi"):                         # the same call again (row pos is rewritten with the same values)
        out = _self_call(L, qkv, Kc, Vc, H, _pos(pos), planes=planes)
        _check_split(out, f.f32)
    print(f"self-attn output planes: rel err {err:.3e}")
    assert err < SELF_BOUND


# ---------------------------------------------------------------------------------------------------------------
# cross-attention over the window's fp16 K / V
# ---------------------------------------------------------------------------------------------------------------
class Scratch:
    """split partials and tickets of stb_decode_cross_attn: tickets start at zero"""

    def __init__(self, L, B, H):
        self.splits = L.lib().stb_decode_cross_splits()
        self.partial = torch.full((B * H * self.splits * 66,), NAN, device="cuda")
        self.tickets = torch.zeros(B * H, dtype=torch.int32, device="cuda")


def _cross_call(L, q, K, V, scratch=None, planes="f32"):
    B, H = K.shape[0], K.shape[1]
    scratch = scratch or Scratch(L, B, H)
    out = Out(B, 64 * H, planes)
    L.check(L.lib().stb_decode_cross_attn(L.ptr(q), L.ptr(K), L.ptr(V), B, H, L.ptr(scratch.partial), L.ptr(scratch.tickets),
                                          L.ptr(out.f32), L.ptr(out.hi), L.ptr(out.lo), L.stream_ptr()))
    torch.cuda.synchronize()
    return out


def _cross_ref(q, K, V):
    """float64 softmax(q . K / 8) V over the 1500 keys, K / V [B][H][T][64] upcast exactly (fp16 or fp32 values)"""
    B, H = K.shape[0], K.shape[1]
    qd = q.double().cpu().view(B, H, 64)
    out = torch.empty(B, H, 64, dtype=torch.float64)
    for b0 in range(0, B, 8):                               # a few sequences at a time: 128 x 6 heads is 0.6 GB in float64
        Kd, Vd = K[b0:b0 + 8].double().cpu(), V[b0:b0 + 8].double().cpu()
        p = (torch.einsum("bhtc,bhc->bht", Kd, qd[b0:b0 + 8]) * SCALE).softmax(-1)
        out[b0:b0 + 8] = torch.einsum("bht,bhtc->bhc", p, Vd)
    return out.view(B, 64 * H)


def _cross_inputs(B, H, seed, sigma=3.0):
    """q ~ N(0, sigma^2) (scores with a standard deviation of ~sigma), fp32 K / V ~ N(0, 1) and their fp16 planes"""
    g = _gen(seed)
    q = torch.randn(B, 64 * H, device="cuda", generator=g) * sigma
    K32 = torch.randn(B, H, T, 64, device="cuda", generator=g)
    V32 = torch.randn(B, H, T, 64, device="cuda", generator=g)
    return q, K32, V32


# every Whisper head count; B = 1 (the tensor map drops the batch dimension), 2, 33, and 128 at a small H
CROSS_CASES = [(6, 128), (6, 1), (8, 33), (12, 2), (16, 1), (20, 2), (20, 33)]


@pytest.mark.parametrize("H,B", CROSS_CASES)
def test_cross_attn_head_counts_vs_fp64(L, H, B):
    q, K32, V32 = _cross_inputs(B, H, seed=H * 1000 + B)
    K, V = K32.half(), V32.half()
    out = _cross_call(L, q, K, V)
    o = out.value()
    err = _rel(o, _cross_ref(q, K, V))
    err32 = _rel(o, _cross_ref(q, K32, V32))               # for the record: what the fp16 K / V cost against fp32 ones
    print(f"cross-attn H={H} B={B}: rel err {err:.3e} (vs unrounded fp32 K / V {err32:.3e})")
    assert err < CROSS_BOUND


@pytest.mark.parametrize("H,B", [(20, 2), (6, 1)])
def test_cross_attn_masks_the_zero_filled_keys(L, H, B):
    """every real score ~ -40 (K = -c q^ + noise): a zero key past 1500 would score 0 and take all the weight, pulling
    the output (V ~ 1 + noise) towards 0"""
    g = _gen(H + B)
    q = torch.randn(B, H, 64, device="cuda", generator=g)
    q = q / q.norm(dim=-1, keepdim=True) * 16.0
    K = (-20.0 / 16.0) * q[:, :, None, :] + 0.3 * torch.randn(B, H, T, 64, device="cuda", generator=g)
    V = 1.0 + 0.5 * torch.randn(B, H, T, 64, device="cuda", generator=g)
    K, V, q = K.half(), V.half(), q.reshape(B, 64 * H).contiguous()
    scores = torch.einsum("bhtc,bhc->bht", K.double(), q.view(B, H, 64).double()) * SCALE
    assert scores.max() < -25
    out = _cross_call(L, q, K, V)
    err = _rel(out.value(), _cross_ref(q, K, V))
    print(f"cross-attn negative scores H={H} B={B} (max score {scores.max().item():.1f}): rel err {err:.3e}")
    assert err < CROSS_BOUND


KSTAR = [0, 95, 96, 191, 192, 1343, 1344, 1439, 1440, 1499]   # both sides of chunk and split edges, first and last key


def test_cross_attn_dominant_key_at_split_edges(L):
    """sequence i has one key k* = KSTAR[i] scoring >= 30 above every other: the output is V[k*]"""
    H, B = 8, len(KSTAR)
    q, K32, V32 = _cross_inputs(B, H, seed=4, sigma=1.0)
    qh = q.view(B, H, 64)
    for i, k in enumerate(KSTAR):
        K32[i, :, k] = qh[i] / qh[i].norm(dim=-1, keepdim=True) ** 2 * (8.0 * 45.0)   # score 45
    K, V = K32.half(), V32.half()
    scores = torch.einsum("bhtc,bhc->bht", K.double(), qh.double()) * SCALE
    top2 = scores.topk(2, dim=-1).values
    assert (top2[..., 0] - top2[..., 1]).min() >= 30
    for i, k in enumerate(KSTAR):
        assert (scores[i].argmax(-1) == k).all()
    out = _cross_call(L, q, K, V)
    o = out.value()
    err = _rel(o, _cross_ref(q, K, V))
    vstar = torch.stack([V[i, :, k] for i, k in enumerate(KSTAR)]).double().cpu().view(B, 64 * H)
    err_v = _rel(o, vstar)
    print(f"cross-attn dominant key at {KSTAR}: rel err {err:.3e} (vs V[k*] {err_v:.3e})")
    assert err < CROSS_BOUND and err_v < CROSS_BOUND


def test_cross_attn_merge_rescales_split_maxima(L):
    """the mass sits in two splits (keys 300 and 1100) whose maxima differ by 2 (both carry weight) and by 20 (the merge must
    scale the second down by e^-20, not add it at par); every other key scores ~ -40"""
    H, gaps = 12, [2.0, 20.0]
    B = len(gaps)
    g = _gen(12)
    qh = torch.randn(B, H, 64, device="cuda", generator=g)
    qh = qh / qh.norm(dim=-1, keepdim=True) * 16.0
    K = (-20.0 / 16.0) * qh[:, :, None, :] + 0.3 * torch.randn(B, H, T, 64, device="cuda", generator=g)
    V = torch.randn(B, H, T, 64, device="cuda", generator=g)
    for b, gap in enumerate(gaps):
        K[b, :, 300] = qh[b] / 256.0 * (8.0 * 5.0)              # score 5
        K[b, :, 1100] = qh[b] / 256.0 * (8.0 * (5.0 - gap))     # score 5 - gap
    K, V, q = K.half(), V.half(), qh.reshape(B, 64 * H).contiguous()
    out = _cross_call(L, q, K, V)
    err = _rel(out.value(), _cross_ref(q, K, V))
    print(f"cross-attn two splits, maxima {gaps} apart: rel err {err:.3e}")
    assert err < CROSS_BOUND


def test_cross_attn_uniform_weights(L):
    """q = 0: every key weighs the same, the output is the mean of V over exactly 1500 keys"""
    H, B = 20, 2
    _, _, V32 = _cross_inputs(B, H, seed=8)
    V32 += 1.0                                               # a mean far from 0: 1536 keys would be off by 2.3 %
    K = torch.randn(B, H, T, 64, device="cuda", generator=_gen(9)).half()
    V = V32.half()
    q = torch.zeros(B, 64 * H, device="cuda")
    out = _cross_call(L, q, K, V)
    mean_v = V.double().cpu().mean(2).view(B, 64 * H)
    err = _rel(out.value(), mean_v)
    print(f"cross-attn q = 0: rel err vs mean of V {err:.3e}")
    assert err < CROSS_BOUND


def test_cross_attn_tickets_and_scratch_across_launches(L):
    """5 launches on one partial / tickets pair, a new q each time: tickets back at 0 after every launch, NaN written into
    the partials between launches never reaches the output; the same inputs give bitwise the same output"""
    H, B = 20, 3
    q, K32, V32 = _cross_inputs(B, H, seed=21)
    K, V = K32.half(), V32.half()
    s = Scratch(L, B, H)
    g = _gen(22)
    first = None
    worst = 0.0
    for i in range(5):
        qi = q if i in (0, 4) else torch.randn(B, 64 * H, device="cuda", generator=g) * 3.0
        s.partial.fill_(NAN)
        out = _cross_call(L, qi, K, V, s)
        assert int(torch.count_nonzero(s.tickets)) == 0, f"tickets not re-armed after launch {i}"
        o = out.value()
        assert torch.isfinite(o).all()
        worst = max(worst, _rel(o, _cross_ref(qi, K, V)))
        if i == 0:
            first = out.f32.clone()
    assert torch.equal(_bits(out.f32), _bits(first)), "identical inputs, different outputs"
    print(f"cross-attn 5 launches on one scratch: worst rel err {worst:.3e}")
    assert worst < CROSS_BOUND


def test_cross_attn_output_planes(L):
    H, B = 16, 2
    q, K32, V32 = _cross_inputs(B, H, seed=31)
    K, V = K32.half(), V32.half()
    f = _cross_call(L, q, K, V, planes="f32")
    err = _rel(f.value(), _cross_ref(q, K, V))
    for planes in ("hi+lo", "hi"):
        _check_split(_cross_call(L, q, K, V, planes=planes), f.f32)
    print(f"cross-attn output planes: rel err {err:.3e}")
    assert err < CROSS_BOUND


@pytest.mark.parametrize("H", [6, 20])
def test_cross_kv_head_major_v_is_the_transposed_vT_plane(L, H):
    """stb_cross_kv(decode_layout=1) writes V head-major [B][H][1500][64] for the decode step: it must be the transpose of
    its own V^T hi plane [B][H][64][1504] bitwise, including the last 64-key tile (1500 = 23 x 64 + 28)"""
    import oracle.whisper_ref as W
    from oracle.whisper_ref.model import ModelDimensions
    from stable_ts_b200.model import from_oracle
    d, B = 64 * H, 2
    dims = ModelDimensions(n_mels=80, n_audio_ctx=T, n_audio_state=d, n_audio_head=H, n_audio_layer=1, n_vocab=51864,
                           n_text_ctx=448, n_text_state=d, n_text_head=H, n_text_layer=1)
    gm = from_oracle(W.build_model(dims, seed=H))
    xa = torch.randn(B * T, d, device="cuda", generator=_gen(H))
    hi = xa.half()
    enc = {"f32": xa.view(B, T, d), "hi": hi, "lo": (xa - hi.float()).half(), "B": B}
    ckv = gm.cross_kv(enc, decode=True).view(torch.float16)
    k_elems, v_elems = B * T * d, B * d * 1504               # per layer: K hi | K lo | V^T hi | V^T lo | V hi head-major
    vT = ckv[2 * k_elems: 2 * k_elems + v_elems].view(B, H, 64, 1504)
    v = ckv[2 * k_elems + 2 * v_elems: 3 * k_elems + 2 * v_elems].view(B, H, T, 64)
    assert torch.isfinite(vT[..., :T]).all()
    assert torch.equal(_bits(v), _bits(vT[..., :T].transpose(-1, -2).contiguous()))


# ---------------------------------------------------------------------------------------------------------------
# whole decode steps to the end of the context
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ragged_run(L):
    """2 decoder layers at d = 384 / H = 6; three windows with prompts of 0, 37 and 223 tokens (initial tokens 2, 40 and 226:
    cache_rows = 448 + 224 = 672); a forced script of ordinary text tokens runs the no-prompt window to its n_ctx stop
    (447 steps: global pos reaches cache_rows - 1)"""
    import oracle.whisper_ref as W
    from oracle import stable_path as SP
    from oracle.whisper_ref.model import ModelDimensions
    from stable_ts_b200.model import from_oracle
    from stable_ts_b200.tokenizer import get_tokenizer
    dims = ModelDimensions(n_mels=80, n_audio_ctx=T, n_audio_state=384, n_audio_head=6, n_audio_layer=1, n_vocab=51864,
                           n_text_ctx=448, n_text_state=384, n_text_head=6, n_text_layer=2)
    model = W.build_model(dims, seed=23)
    gm = from_oracle(model)
    tk = get_tokenizer(gm, language="en", task="transcribe", synthetic=True)
    g = torch.Generator().manual_seed(24)
    prompts = [[], torch.randint(300, 40000, (37,), generator=g).tolist(), torch.randint(300, 40000, (223,), generator=g).tolist()]
    audios = torch.stack([SP.synth_audio(480000, seed=240 + i) for i in range(3)])
    steps = dims.n_text_ctx
    script = SP.synth_token_script(steps, tk.eot, seed=25)
    return dict(SP=SP, model=model, gm=gm, tk=tk, prompts=prompts, audios=audios, steps=steps, script=script, refs=[])


def _run_ragged(r, rep, reuse_buffers=False):
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    gm, B = r["gm"], 3 * rep
    enc = gm.encode(gm.log_mel(r["audios"].repeat(rep, 1).cuda()))
    opt = DecodingOptions(language="en", sample_len=r["steps"], without_timestamps=True)
    forced = torch.tensor(r["script"])[:, None].repeat(1, B)
    _, x = decode_windows(gm, r["tk"], enc, opt, forced_tokens=forced, return_step_logits=True, prompts=r["prompts"] * rep,
                          reuse_buffers=reuse_buffers)
    return enc, x


def _step_refs(r, feats, j):
    """float64 step logits of the oracle's decode of window j % 3 on these encoder features (shared by equal inputs)"""
    import copy
    import torch.nn.functional as F
    from oracle.whisper_ref import model as WM
    p = r["prompts"][j % 3]
    ref = next((s for w, a, s in r["refs"] if w == j % 3 and torch.equal(a, feats)), None)
    if ref is None:
        if "m64" not in r:
            r["m64"] = copy.deepcopy(r["model"]).double()
        with pytest.MonkeyPatch.context() as mp:
            # the oracle's LayerNorm computes in fp32 (a guard for fp16 models); in the float64 model it keeps float64
            mp.setattr(WM.LayerNorm, "forward", lambda self, x: F.layer_norm(x, self.normalized_shape, self.weight, self.bias, self.eps))
            _, _, ex = r["SP"].decode_window(r["m64"], torch.zeros(80, 3000), audio_features=feats[None], forced_tokens=r["script"],
                                             return_step_logits=True, sample_len=r["steps"], language="en",
                                             without_timestamps=True, prompt=p or None)
        ref = ex["step_logits"]
        r["refs"].append((j % 3, feats, ref))
    return ref


@pytest.mark.parametrize("rep", [1, 7])
def test_step_logits_to_the_end_of_the_context_vs_fp64(ragged_run, rep):
    """B = 3 (GEMV linears) and B = 21 (cluster linears): every step each window ran, against the float64 oracle"""
    r = ragged_run
    enc, x = _run_ragged(r, rep)
    B = 3 * rep
    feats = enc["f32"].view(B, T, -1).cpu().double()
    n_steps = []
    worst = 0.0
    for j in range(B):
        ref = _step_refs(r, feats[j], j)
        n_steps.append(len(ref))
        assert len(ref) <= len(x["step_logits"])
        for i, rl in enumerate(ref):
            rl, gl = rl.double(), x["step_logits"][i][j].double().cpu()
            fin = rl > -1e30
            assert torch.equal(fin, gl > -1e30), f"mask mismatch, window {j} step {i}"
            worst = max(worst, ((gl[fin] - rl[fin]).abs().max() / rl[fin].abs().max()).item())
    assert n_steps[:3] == [447, 409, 223], n_steps          # the no-prompt window reaches its n_ctx stop
    print(f"B={B}: ragged prompts to the end of the context, worst step-logit rel err {worst:.2e}")
    assert worst < STEP_BOUND


def test_stale_model_owned_cache_is_never_read(ragged_run):
    """reuse_buffers=True on a model-owned K/V cache full of 0xFF bytes (NaN): the same step logits, bitwise"""
    from stable_ts_b200 import _lib
    r = ragged_run
    gm = r["gm"]
    _, fresh = _run_ragged(r, 1)
    nbytes = _lib.lib().stb_decode_state_bytes_rows(gm._h, 3, 448 + 224)
    gm._buf("decode_state", nbytes).fill_(0xFF)
    _, stale = _run_ragged(r, 1, reuse_buffers=True)
    assert len(fresh["step_logits"]) == len(stale["step_logits"]) == 447
    for a, b in zip(fresh["step_logits"], stale["step_logits"]):
        assert torch.equal(_bits(a), _bits(b))
