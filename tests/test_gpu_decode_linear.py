"""GPU tests of the decode-step cluster linear (stb_decode_linear, csrc/decode_linear.cu) against float64 references computed
on the CPU: every batch tile width with idle and partial cluster ranks, every cluster size, each epilogue on its own, the
rows and columns the kernel must leave alone, and bit-reproducibility.

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


def _call(L, x, W, N, out, passes=3, bias=None, act=0, res=None, ld_res=0):
    """x: (hi, lo) planes [B][K] or an fp32 matrix to split; W: (hi, lo) planes [N][K] or fp32"""
    xh, xl = x if isinstance(x, tuple) else _split(x, passes == 3)
    wh, wl = W if isinstance(W, tuple) else _split(W, passes == 3)
    B, K = xh.shape
    L.check(L.lib().stb_decode_linear(L.ptr(xh), L.ptr(xl), B, K, L.ptr(wh), L.ptr(wl), N, L.ptr(bias), act, L.ptr(res),
                                      ld_res, L.ptr(out.f32), L.ptr(out.hi), L.ptr(out.lo), out.ld, L.stream_ptr()))
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
# the q/k/v projection of large-v3 at 48 sequences also runs on LayerNorm-ed residual-stream rows (_layernormed_rows)
LAYERNORMED_SHAPE = (48, 3840, 1280)


def _layernormed_rows(B, d, seed):
    """float64 LayerNorm (random gamma / beta) of residual-stream rows with mean/std 0, 3, 10, 100 (B // 5 rows each) and of
    rows with two features at 50 sigma, as fp32: what the decode step feeds a Linear after a LayerNorm, outliers included.
    Returns the rows and {group name: row indices}."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, d, device="cuda", generator=g)
    groups, per = {}, B // 5
    for i, r in enumerate((0, 3, 10, 100)):
        x[i * per: (i + 1) * per] += r
        groups[f"mean/std {r}"] = list(range(i * per, (i + 1) * per))
    spikes = list(range(4 * per, B))
    x[spikes, 7] = 50.0
    x[spikes, d - 3] = -50.0
    groups["two features at 50 sigma"] = spikes
    gamma = 1.0 + 0.1 * torch.randn(d, device="cuda", generator=g)
    beta = 0.1 * torch.randn(d, device="cuda", generator=g)
    x = x.double()
    mu = x.mean(1, keepdim=True)
    var = ((x - mu) ** 2).mean(1, keepdim=True)
    return ((x - mu) / torch.sqrt(var + 1e-5) * gamma.double() + beta.double()).float(), groups


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
    if (B, n, k) == LAYERNORMED_SHAPE:                         # per row group, relative to the group's largest value
        X, groups = _layernormed_rows(B, k, 42)
        bias = 0.1 * torch.randn(n, device="cuda", generator=torch.Generator(device="cuda").manual_seed(43))
        out = Out(n, ld)
        _call(L, X, W, n, out, passes, bias=bias)
        out.check_guards(B)
        D, R = out.value(B), _ref(X, Wd, bias)
        for name, rows in groups.items():
            err = _rel(D[rows], R[rows])
            print(f"  LayerNorm-ed rows, {name}: rel err {err:.3e}")
            assert err < _bound(k, passes), name


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
    """Fixed summation order over the cluster's ranks: two identical calls, identical bits."""
    for B, n, k in [(65, 3840, 1280), (48, 1280, 5120), (17, 1002, 1280)]:
        W, _ = _weights(n, k)
        X = _x(B, k, 77)
        bias = torch.randn(n, device="cuda")
        res = torch.randn(B, n, device="cuda")
        outs = []
        for _ in range(2):
            out = Out(n, (n + 3) // 4 * 4, hi=True, lo=True)
            _call(L, X, W, n, out, bias=bias, act=1, res=res, ld_res=n)
            outs.append(out.planes())
        for a, b in zip(*outs):
            assert torch.equal(_bits(a), _bits(b)), (B, n, k)
