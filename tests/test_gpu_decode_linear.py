"""GPU tests of the decode-step cluster linear (stb_decode_linear, csrc/decode_linear.cu) against float64 references computed
on the CPU: every batch tile width with idle and partial cluster ranks, every cluster size, each epilogue on its own, the
rows and columns the kernel must leave alone, bit-reproducibility, the per-tile row statistics it leaves for the next
Linear, and the LayerNorm folded into the decode step's linears (kernel level and end to end).

Run on an H100:  python -m pytest tests/test_gpu_decode_linear.py -q -s
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")
MAX_B = 128                       # largest batch the kernel takes: every output plane is allocated this tall


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from stable_ts_b200 import _lib
    _lib.lib()
    return _lib


def _split(x, lo=True):
    hi = x.half()
    return hi, ((x - hi.float()).half() if lo else None)


def _bound(K, passes):
    """relative to max|ref|: the bound of the GEMV decode linear (test_gpu_kernels.py), ~sqrt(K) growth for three passes"""
    return max(3e-6, 4e-7 * K ** 0.5) if passes == 3 else 3e-3


def _rel(D, R):
    return ((D.double().cpu() - R).abs().max() / R.abs().max()).item()


_W = {}


def _weights(n, k):
    """seeded W [n][k] (fp32, cuda) and its float64 copy on the CPU, cached: the vocabulary matrix is 0.5 GB in float64"""
    if (n, k) not in _W:
        g = torch.Generator(device="cuda").manual_seed(n * 7 + k)
        W = torch.randn(n, k, device="cuda", generator=g) * (1.0 / k ** 0.5)
        _W[(n, k)] = (W, W.double().cpu())
    return _W[(n, k)]


class Out:
    """Output planes of MAX_B rows x ld columns filled with NaN: whatever the kernel must not write stays NaN."""

    def __init__(self, N, ld, f32=True, hi=False, lo=False):
        self.N, self.ld = N, ld
        self.f32 = torch.full((MAX_B, ld), NAN, device="cuda") if f32 else None
        self.hi = torch.full((MAX_B, ld), NAN, dtype=torch.float16, device="cuda") if hi else None
        self.lo = torch.full((MAX_B, ld), NAN, dtype=torch.float16, device="cuda") if lo else None

    def planes(self):
        return [p for p in (self.f32, self.hi, self.lo) if p is not None]

    def value(self, B):
        """what was computed for rows < B, columns < N, as float64 on the CPU"""
        if self.f32 is not None:
            return self.f32[:B, : self.N].double().cpu()
        v = self.hi[:B, : self.N].double()
        if self.lo is not None:
            v = v + self.lo[:B, : self.N].double()
        return v.cpu()

    def check_guards(self, B):
        for p in self.planes():
            assert not torch.isnan(p[:B, : self.N]).any(), "an output element was not written"
            assert torch.isnan(p[B:]).all(), f"rows >= B = {B} were written"
            assert torch.isnan(p[:B, self.N:]).all(), f"columns [N, ld_out) = [{self.N}, {self.ld}) were written"


def _call(L, x, W, N, out, passes=3, bias=None, act=0, res=None, ld_res=0, stats_in=None, tiles_in=0, features=0, wsum=None,
          stats_out=None):
    """x: (hi, lo) planes [B][K] or an fp32 matrix to split; W: (hi, lo) planes [N][K] or fp32"""
    xh, xl = x if isinstance(x, tuple) else _split(x, passes == 3)
    wh, wl = W if isinstance(W, tuple) else _split(W, passes == 3)
    B, K = xh.shape
    L.check(L.lib().stb_decode_linear(L.ptr(xh), L.ptr(xl), B, K, L.ptr(wh), L.ptr(wl), N, L.ptr(bias), act, L.ptr(res),
                                      ld_res, L.ptr(out.f32), L.ptr(out.hi), L.ptr(out.lo), out.ld, L.ptr(stats_in), tiles_in,
                                      features, L.ptr(wsum), L.ptr(stats_out), L.stream_ptr()))
    torch.cuda.synchronize()


def _ref(X, Wd, bias=None, act=0, res=None):
    D = X.double().cpu() @ Wd.T
    if bias is not None:
        D = D + bias.double().cpu()
    if act == 1:
        D = torch.nn.functional.gelu(D)
    if res is not None:
        D = D + res.double().cpu()
    return D


def _x(B, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B, K, device="cuda", generator=g)


# the Linears of large-v3 (d = 1280: q/k/v, out, fc1, fc2, vocabulary) and tiny (d = 384), plus n = 130 (last tile: 2
# features); B covers BN = 32 / 64 / 128, batches that fill a tile and ones that spill into the next, and cluster ranks
# that own part of a tile or none of it (B = 48 at split 8: ranks 6 and 7)
SHAPES = [(1, 1280, 1280), (17, 3840, 1280), (32, 5120, 1280), (33, 1280, 5120), (48, 1280, 1280), (48, 3840, 1280),
          (48, 5120, 1280), (48, 1280, 5120), (48, 51866, 1280), (64, 384, 384), (65, 3840, 1280), (127, 1280, 1280),
          (128, 1280, 5120), (128, 51866, 1280), (128, 384, 384), (17, 130, 384), (65, 130, 1280), (1, 51866, 1280)]


@pytest.mark.parametrize("B,n,k", SHAPES)
@pytest.mark.parametrize("passes", [3, 1])
def test_decode_linear_vs_fp64(L, B, n, k, passes):
    W, Wd = _weights(n, k)
    X = _x(B, k, B * 131 + n + k)
    ld = (n + 3) // 4 * 4 + 4
    out = Out(n, ld)
    _call(L, X, W, n, out, passes)
    out.check_guards(B)
    err = _rel(out.value(B), _ref(X, Wd))
    split = L.lib().stb_decode_linear_split(n, k)
    print(f"decode_linear B={B} n={n} k={k} split={split} passes={passes}: rel err {err:.3e}")
    assert err < _bound(k, passes)


def _cluster_cases(L):
    """(n, k) per cluster size 1..8 on this device, found by asking the library; uneven k-block partitions preferred"""
    best = {}
    for mt in range(1, 129):
        for nkb in (1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 17, 20):
            n, k = 128 * mt, 64 * nkb
            s = L.lib().stb_decode_linear_split(n, k)
            assert 1 <= s <= 8 and s <= nkb, (n, k, s)
            key = (nkb % s == 0, n * k)
            if s not in best or key < best[s][0]:
                best[s] = (key, n, k)
    return {s: (n, k) for s, (_, n, k) in best.items()}


def test_every_cluster_size(L):
    """Cluster sizes 1..8 each run at least once (the model shapes of one device reach only a few of them), several with a
    k-block count the size does not divide, plus a ragged n; B = 48 leaves the last ranks of a split-8 cluster idle."""
    assert L.lib().stb_decode_linear_split(130, 100) == 0 and b"n=130 k=100" in L.lib().stb_last_error()
    cases = _cluster_cases(L)
    print(f"cluster sizes reached: {sorted(cases)}  (n, k): {[cases[s] for s in sorted(cases)]}")
    assert sorted(cases) == list(range(1, 9))
    uneven = [s for s, (n, k) in cases.items() if (k // 64) % s != 0]
    assert uneven, "no case with an uneven k-block partition"
    runs = [(s, n, k) for s, (n, k) in sorted(cases.items())] + [(L.lib().stb_decode_linear_split(1000, 640), 1000, 640)]
    for s, n, k in runs:
        W, Wd = _weights(n, k)
        for B in (48, 128):
            X = _x(B, k, s * 1000 + B)
            bias = torch.randn(n, device="cuda")
            out = Out(n, (n + 3) // 4 * 4 + 4)
            _call(L, X, W, n, out, bias=bias, act=1)
            out.check_guards(B)
            err = _rel(out.value(B), _ref(X, Wd, bias=bias, act=1))
            print(f"  split={s} n={n} k={k} (k blocks {k // 64}) B={B}: rel err {err:.3e}")
            assert err < _bound(k, 3)


def test_epilogues_one_at_a_time(L):
    """bias, GELU, residual (also in place, as the decode step updates its residual stream), split outputs with and without
    the lo plane, fp32 and split together (bit-consistent), the scalar store path and residual pitches != output pitch.
    N = 1002: the last feature quad is partial; B = 37 at split 8: rank 4 owns a partial slice, ranks 5..7 none."""
    B, N, K = 37, 1002, 1280
    W, Wd = _weights(N, K)
    X = _x(B, K, 5)
    g = torch.Generator(device="cuda").manual_seed(6)
    bias = torch.randn(N, device="cuda", generator=g)
    bound = _bound(K, 3)
    ld = 1008

    def res_with(ld_res):
        r = torch.full((B, ld_res), NAN, device="cuda")
        r[:, :N] = torch.randn(B, N, device="cuda", generator=g)
        return r

    def run(name, out, tol=bound, **kw):
        _call(L, X, W, N, out, **kw)
        out.check_guards(B)
        res = kw.get("res")
        R = _ref(X, Wd, kw.get("bias"), kw.get("act", 0), None if res is None else res[:B, :N])
        err = _rel(out.value(B), R)
        print(f"epilogue {name}: rel err {err:.3e}")
        assert err < tol, name
        return R

    run("bias", Out(N, ld), bias=bias)
    run("bias + gelu", Out(N, ld), bias=bias, act=1)
    r = res_with(ld)
    run("bias + residual", Out(N, ld), bias=bias, res=r, ld_res=ld)
    run("bias + gelu + residual", Out(N, ld), bias=bias, act=1, res=r, ld_res=ld)
    # residual in place: res is out_f32
    out = Out(N, ld)
    out.f32[:B, :N] = r[:, :N]
    _call(L, X, W, N, out, bias=bias, res=out.f32, ld_res=ld)
    out.check_guards(B)
    err = _rel(out.value(B), _ref(X, Wd, bias, 0, r[:, :N]))
    print(f"epilogue residual in place: rel err {err:.3e}")
    assert err < bound
    run("split hi + lo", Out(N, ld, f32=False, hi=True, lo=True), bias=bias, act=1)
    run("split hi only", Out(N, ld, f32=False, hi=True), tol=2.0 ** -11 + bound, bias=bias, act=1)
    # fp32 and split together: the planes are exactly the fp16 split of the fp32 values
    for ld_out in (ld, N + 3):                                # vector and scalar store paths
        out = Out(N, ld_out, hi=True, lo=True)
        run(f"fp32 + split, ld_out={ld_out}", out, bias=bias, act=1, res=r, ld_res=ld)
        f, hi, lo = out.f32[:B, :N], out.hi[:B, :N], out.lo[:B, :N]
        assert torch.equal(hi, f.half()) and torch.equal(lo, (f - hi.float()).half())
    # residual pitch != output pitch, a multiple of 4 (vector loads) and not (scalar loads)
    for ld_res in (1012, 1005):
        r2 = res_with(ld_res)
        run(f"ld_res={ld_res}, ld_out={ld}", Out(N, ld), bias=bias, act=1, res=r2, ld_res=ld_res)
    run(f"ld_res={ld}, ld_out={N + 3}", Out(N, N + 3), bias=bias, res=r, ld_res=ld)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16)


def test_bit_reproducible(L):
    """Fixed summation order over the cluster's ranks and in every warp reduction: two identical calls, identical bits."""
    for B, n, k in [(65, 3840, 1280), (48, 1280, 5120), (17, 1002, 1280)]:
        W, _ = _weights(n, k)
        X = _x(B, k, 77)
        bias = torch.randn(n, device="cuda")
        res = torch.randn(B, n, device="cuda")
        outs = []
        for _ in range(2):
            out = Out(n, (n + 3) // 4 * 4, hi=True, lo=True)
            stats = torch.full(((n + 127) // 128, B, 2), NAN, device="cuda")
            _call(L, X, W, n, out, bias=bias, act=1, res=res, ld_res=n, stats_out=stats)
            outs.append([*out.planes(), stats])
        for a, b in zip(*outs):
            assert torch.equal(_bits(a), _bits(b)), (B, n, k)


def _tile_stats(Y, features):
    """float64 per-128-feature-tile (sum, sum of squares about the tile mean) of rows Y [B][features] -> [tiles][B][2]"""
    out = []
    for t0 in range(0, features, 128):
        v = Y[:, t0: min(t0 + 128, features)]
        s = v.sum(1)
        m2 = ((v - (s / v.shape[1])[:, None]) ** 2).sum(1)
        out.append(torch.stack([s, m2], 1))
    return torch.stack(out, 0)


@pytest.mark.parametrize("B,N", [(48, 1002), (65, 130), (21, 1280)])
def test_stats_out_per_tile(L, B, N):
    """stats_out: per 128-feature tile and sequence, the sum and the sum of squared deviations from the tile mean of the
    FINAL values (after bias, GELU and residual); ragged last tiles (106 and 2 features).  Rows offset by 100x their spread
    as well: the statistics must not lose the spread to cancellation."""
    K = 1280
    W, Wd = _weights(N, K)
    X = _x(B, K, B + N)
    bias = torch.randn(N, device="cuda")
    res = torch.randn(B, N, device="cuda") + torch.linspace(-100, 100, B, device="cuda")[:, None]
    tiles = (N + 127) // 128
    for kw in (dict(bias=bias, act=1), dict(bias=bias, act=1, res=res, ld_res=N)):
        out = Out(N, (N + 3) // 4 * 4)
        st = torch.full((tiles, B, 2), NAN, device="cuda")
        _call(L, X, W, N, out, stats_out=st, **kw)
        got = st.double().cpu()
        assert not torch.isnan(got).any()
        mine = _tile_stats(out.value(B), N)                   # of the values the kernel stored
        R = _ref(X, Wd, kw["bias"], kw["act"], kw.get("res"))
        ref = _tile_stats(R, N)                               # of the exact values
        # sums relative to the sum of magnitudes; M2 relative to itself, floored at one unit of variance (the scale of the
        # data) per feature: a 2-feature tile can have a tiny M2
        abs_sum = torch.stack([R[:, t0: t0 + 128].abs().sum(1) for t0 in range(0, N, 128)], 0)
        floor = torch.tensor([min(128, N - t0) for t0 in range(0, N, 128)], dtype=torch.float64)[:, None]
        e_sum = ((got[..., 0] - mine[..., 0]).abs() / abs_sum).max().item()
        e_m2 = ((got[..., 1] - mine[..., 1]).abs() / torch.maximum(mine[..., 1], floor)).max().item()
        r_sum = ((got[..., 0] - ref[..., 0]).abs() / abs_sum).max().item()
        r_m2 = ((got[..., 1] - ref[..., 1]).abs() / torch.maximum(ref[..., 1], floor)).max().item()
        print(f"stats_out B={B} N={N} residual={'res' in kw}: vs stored values sum {e_sum:.2e} m2 {e_m2:.2e}; "
              f"vs fp64 sum {r_sum:.2e} m2 {r_m2:.2e}")
        assert e_sum < 1e-5 and e_m2 < 1e-5
        assert r_sum < 5e-5 and r_m2 < 2e-4


def _layernorm64(Y, gamma, beta):
    Y = Y.double()
    mu = Y.mean(1, keepdim=True)
    var = ((Y - mu) ** 2).mean(1, keepdim=True)
    return (Y - mu) / torch.sqrt(var + 1e-5) * gamma.double().cpu() + beta.double().cpu()


RATIOS = (0, 3, 10, 100)


def _offset_rows(B, d, seed):
    """residual-stream rows with mean/std 0, 3, 10, 100 (B // 5 rows each) and rows with two features at 50 sigma"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, d, device="cuda", generator=g)
    groups, per = {}, B // 5
    for i, r in enumerate(RATIOS):
        x[i * per: (i + 1) * per] += r
        groups[f"mean/std {r}"] = list(range(i * per, (i + 1) * per))
    spikes = list(range(len(RATIOS) * per, B))
    x[spikes, 7] = 50.0
    x[spikes, d - 3] = -50.0
    groups["two features at 50 sigma"] = spikes
    return x, groups


def test_folded_layernorm_chain_vs_fp64(L):
    """The decode step's folded LayerNorm, as the step runs it: a producer Linear with a residual (the out / fc2 projection)
    leaves its output as split planes plus per-tile statistics; the consumer (q/k/v) runs on the RAW rows with W diag(gamma)
    planes and the fold vector (fold_layernorm_into_linear, as the model packs them) and applies the LayerNorm in its
    epilogue.  Against float64 LayerNorm(producer output) W^T + b, for rows far from zero mean.  Printed beside: LayerNorm in
    float64, then the same kernel on the normalised rows (the unfused route's error)."""
    from stable_ts_b200.model import fold_layernorm_into_linear
    B, d, n2 = 48, 1280, 3840
    g = torch.Generator(device="cuda").manual_seed(41)
    A = torch.randn(B, d, device="cuda", generator=g)                     # the attention output feeding the producer
    Wo = torch.randn(d, d, device="cuda", generator=g) * 0.005
    bo = torch.randn(d, device="cuda", generator=g) * 0.01
    res, groups = _offset_rows(B, d, 42)
    W2, W2d = _weights(n2, d)
    b2 = torch.randn(n2, device="cuda", generator=g) * 0.1
    gamma = 1.0 + 0.1 * torch.randn(d, device="cuda", generator=g)
    beta = 0.1 * torch.randn(d, device="cuda", generator=g)
    Y = _ref(A, Wo.double().cpu(), bo, 0, res)                           # producer output, exact
    R = _layernorm64(Y, gamma, beta) @ W2d.T + b2.double().cpu()
    sd = (Y - Y.mean(1, keepdim=True)).pow(2).mean(1).sqrt()
    report = {}
    for passes in (3, 1):
        lo = passes == 3
        prod = Out(d, d, hi=True, lo=lo)
        stats = torch.full((d // 128, B, 2), NAN, device="cuda")
        _call(L, A, Wo, d, prod, passes, bias=bo, res=res, ld_res=d, stats_out=stats)
        hi, lo_p, fold = fold_layernorm_into_linear(W2, b2, gamma, beta, lo)
        n_pad = fold.shape[1]
        cons = Out(n2, n2)
        _call(L, (prod.hi[:B], prod.lo[:B] if lo else None), (hi, lo_p), n2, cons, passes, bias=fold[1], stats_in=stats,
              tiles_in=d // 128, features=d, wsum=fold[0])
        cons.check_guards(B)
        assert n_pad % 4 == 0
        # the same folded call with exact whole-row statistics of the stored producer output: what is left is the GEMM's
        # own error on the un-centred rows (fp32 accumulation of the mean's share, mean x rowsum(W') ~ 100 x the result at
        # mean/std 100), which no statistics can remove
        Ys = prod.f32[:B].double().cpu()
        exact = torch.stack([Ys.sum(1), ((Ys - Ys.mean(1, keepdim=True)) ** 2).sum(1)], 1)[None].float().cuda()
        ex = Out(n2, n2)
        _call(L, (prod.hi[:B], prod.lo[:B] if lo else None), (hi, lo_p), n2, ex, passes, bias=fold[1], stats_in=exact,
              tiles_in=1, features=d, wsum=fold[0])
        # unfused route: LayerNorm in float64 of the producer's stored output, then the same kernel on the normalised rows
        ln = _layernorm64(Ys, gamma, beta).float().cuda()
        un = Out(n2, n2)
        _call(L, ln, W2, n2, un, passes, bias=b2)
        for name, rows in groups.items():
            Rg = R[rows]
            ef, ee, eu = (((o.value(B)[rows] - Rg).abs().max() / Rg.abs().max()).item() for o in (cons, ex, un))
            ratio = (Y[rows].mean(1).abs() / sd[rows]).max().item()
            report[(passes, name)] = (ef, ee, eu)
            print(f"folded LayerNorm {'fp16x3' if lo else 'fp16'} {name} (max mean/std {ratio:.1f}): folded {ef:.2e}, "
                  f"folded with exact statistics {ee:.2e}, fp64 LayerNorm + same kernel {eu:.2e}")
    for name in groups:
        ef, ee, _ = report[(3, name)]
        # the statistics the producer left cost at most a quarter on top of the GEMM's own error
        assert ef < (2e-4 if name == "mean/std 100" else 2e-5) and ef < 1.25 * ee + 1e-6, name
    for name in groups:                                       # the unfused one-pass route: the GEMM bound of its K
        assert report[(1, name)][2] < _bound(d, 1), name


def _offset_model(precision):
    """d = 384 decoder whose positional embedding is shifted by 10x its row std: every residual-stream row of the step,
    from the embedding on, sits far from zero mean"""
    import oracle.whisper_ref as W
    from oracle.whisper_ref.model import ModelDimensions
    from stable_ts_b200.model import from_oracle
    from stable_ts_b200.tokenizer import get_tokenizer
    dims = ModelDimensions(n_mels=80, n_audio_ctx=1500, n_audio_state=384, n_audio_head=6, n_audio_layer=1, n_vocab=51864,
                           n_text_ctx=448, n_text_state=384, n_text_head=6, n_text_layer=2)
    model = W.build_model(dims, seed=51)
    with torch.no_grad():
        pe = model.decoder.positional_embedding
        pe += 10.0 * pe.std(dim=1, keepdim=True)
    gm = from_oracle(model, precision=precision)
    tk = get_tokenizer(gm, language="en", task="transcribe", synthetic=True)
    return gm, tk


def _step_logits_on_off(gm, tk, B):
    from oracle import stable_path as SP
    from stable_ts_b200 import _lib as L
    from stable_ts_b200.decode import DecodingOptions, decode_windows
    audios = torch.stack([SP.synth_audio(480000, seed=600 + i) for i in range(3)]).repeat(B // 3, 1)
    enc = gm.encode(gm.log_mel(audios.cuda()))
    opt = DecodingOptions(sample_len=8)
    default = L.get_option("decode_fused_ln")
    try:
        L.set_option("decode_fused_ln", 0)
        r0, x0 = decode_windows(gm, tk, enc, opt, return_step_logits=True)
        L.set_option("decode_fused_ln", 1)
        r1, x1 = decode_windows(gm, tk, enc, opt, return_step_logits=True)
    finally:
        L.set_option("decode_fused_ln", default)
    return r0, x0["step_logits"], r1, x1["step_logits"]


def test_folded_layernorm_step_with_offset_rows():
    """End to end at B = 21 (cluster route, BN = 32): step logits with the LayerNorms folded into the linears (statistics
    from embed_step and from every producer Linear) agree with the LayerNorm kernels' within 2e-5, and the tokens are equal."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    gm, tk = _offset_model("fp16x3")
    r0, x0, r1, x1 = _step_logits_on_off(gm, tk, 21)
    worst = 0.0
    for a, b in zip(x0, x1):
        a, b = a.float().cpu(), b.float().cpu()
        fin = a > -1e30
        assert torch.equal(fin, b > -1e30)
        worst = max(worst, ((a[fin] - b[fin]).abs().max() / a[fin].abs().max()).item())
    print(f"offset rows, B=21: folded LayerNorm vs LayerNorm kernels, worst step-logit rel diff {worst:.2e}")
    assert worst < 2e-5
    for a, b in zip(r0, r1):
        assert a.tokens == b.tokens


def test_fp16_model_ignores_folded_layernorm():
    """In STB_PREC_FP16 the folded route would feed the raw, un-centred row through one fp16 plane (error ~ 2^-11 mean/std
    after centring instead of 2^-11): an fp16 model packs no fold tensors and its step is the same with the option on."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    gm, tk = _offset_model("fp16")
    assert not gm.fold_layernorm
    r0, x0, r1, x1 = _step_logits_on_off(gm, tk, 21)
    for a, b in zip(x0, x1):
        assert torch.equal(a, b)
    for a, b in zip(r0, r1):
        assert a.tokens == b.tokens
