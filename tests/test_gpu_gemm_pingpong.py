"""stb_gemm's persistent kernel, where its two consumer warpgroups take turns over whole tiles, against float64: tile counts
that leave a consumer idle or give one an extra tile, every tile width, every epilogue on shapes with several tiles per
consumer, the head-major column mapping of the cross-attention K projection, and run-to-run bitwise stability."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from stable_ts_b200 import _lib
    _lib.lib()
    return _lib


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _split(x, lo=True):
    hi = x.half()
    return hi, ((x - hi.float()).half() if lo else None)


def _run(L, A, B, passes=3, bias=None, act=0, residual=None, alpha=1.0, out="f32", transposed=False, in_place=False):
    """A [M,K], B [N,K] fp32 cuda -> D via stb_gemm; out is "f32", "split" or "both" (fp32 and split planes at once)"""
    M, K = A.shape
    N = B.shape[0]
    ah, al = _split(A, passes == 3)
    bh, bl = _split(B, passes == 3)
    opa = L.Operand(L.ptr(ah), L.ptr(al), M, K, K, 0, 0)
    opb = L.Operand(L.ptr(bh), L.ptr(bl), N, K, K, 0, 0)
    rows, ld = (N, M) if transposed else (M, N)
    ldp = (ld + 7) // 8 * 8
    of = torch.full((rows, ldp), float("nan"), device="cuda") if out in ("f32", "both") else None
    if in_place:
        of[:, :ld] = residual
    oh = torch.full((rows, ldp), float("nan"), dtype=torch.float16, device="cuda") if out in ("split", "both") else None
    ol = torch.full_like(oh, float("nan")) if oh is not None else None
    ep = L.Epilogue()
    ep.out_f32, ep.out_hi, ep.out_lo = L.ptr(of), L.ptr(oh), L.ptr(ol)
    ep.ld_out = ldp
    ep.transposed = int(transposed)
    ep.bias = L.ptr(bias)
    res = of if in_place else residual
    ep.residual = L.ptr(res)
    ep.ld_res = res.stride(0) if res is not None else 0
    ep.alpha = alpha
    ep.act = act
    L.check(L.lib().stb_gemm(ctypes.byref(opa), ctypes.byref(opb), 1, 1, ctypes.byref(ep), L.stream_ptr()))
    torch.cuda.synchronize()
    f = of[:, :ld].double().cpu() if of is not None else None
    s = (oh[:, :ld].double() + ol[:, :ld].double()).cpu() if oh is not None else None
    return f, s


def _ref(A, B, bias=None, act=0, residual=None, alpha=1.0):
    D = alpha * (A.double().cpu() @ B.double().cpu().T)
    if bias is not None:
        D = D + bias.double().cpu()
    if act == 1:
        D = torch.nn.functional.gelu(D)
    if residual is not None:
        D = D + residual.double().cpu()
    return D


def _rel(D, R):
    assert torch.isfinite(D).all()
    return (D - R).abs().max().item() / R.abs().max().item()


def _inputs(M, N, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(M, K, device="cuda", generator=g), torch.randn(N, K, device="cuda", generator=g) * 0.3


@pytest.mark.parametrize("which", ["one", "sms-1", "sms+1", "2sms+1"])
def test_tile_counts_idle_and_extra_consumer(L, which):
    """128 x 128 tiles, one n block: the tile count is the number of 128-row blocks (the last one ragged)"""
    sms = _sms()
    tiles = {"one": 1, "sms-1": sms - 1, "sms+1": sms + 1, "2sms+1": 2 * sms + 1}[which]
    M, N, K = 128 * (tiles - 1) + 77, 128, 192
    A, B = _inputs(M, N, K, tiles)
    D, _ = _run(L, A, B)
    err = _rel(D, _ref(A, B))
    print(f"{tiles} tiles ({sms} SMs): rel err {err:.3e}")
    assert err < 3e-6


@pytest.mark.parametrize("N", [16, 32, 64, 128])
@pytest.mark.parametrize("passes", [3, 1])
def test_every_tile_width_several_tiles_per_consumer(L, N, passes):
    """N picks the tile width (BN = 16 / 32 / 64 / 128); 8 tiles per SM or more, so each consumer runs 4 or more"""
    M, K = 128 * 8 * _sms() + 33, 320
    A, B = _inputs(M, N, K, N + passes)
    D, _ = _run(L, A, B, passes)
    err = _rel(D, _ref(A, B))
    print(f"BN {N} passes {passes} M {M}: rel err {err:.3e}")
    assert err < (3e-6 if passes == 3 else 3e-3)


EPILOGUES = {
    "bias": dict(bias=True),
    "gelu": dict(bias=True, act=1),
    "residual_in_place": dict(bias=True, residual=True, in_place=True),
    "alpha": dict(alpha=0.125),
    "split": dict(bias=True, act=1, out="split"),
    "f32_and_split": dict(bias=True, residual=True, out="both"),
    "transposed_split": dict(bias=True, out="split", transposed=True),
    "transposed_f32": dict(alpha=0.5, transposed=True),
}


@pytest.mark.parametrize("name", list(EPILOGUES))
def test_epilogues_multi_tile(L, name):
    """every epilogue on 1.5 tiles per consumer or more (odd N: the last column pair of every row is a single column)"""
    kw = dict(EPILOGUES[name])
    M, N, K = 128 * 3 * _sms() + 5, 263, 448
    A, B = _inputs(M, N, K, 7)
    g = torch.Generator(device="cuda").manual_seed(8)
    bias = torch.randn(N, device="cuda", generator=g) if kw.pop("bias", False) else None
    res = torch.randn(M, N, device="cuda", generator=g) if kw.pop("residual", False) else None
    out = kw.get("out", "f32")
    f, s = _run(L, A, B, 3, bias=bias, residual=res, **kw)
    R = _ref(A, B, bias=bias, act=kw.get("act", 0), residual=res, alpha=kw.get("alpha", 1.0))
    if kw.get("transposed"):
        R = R.T
    for D in (f, s):
        if D is not None:
            err = _rel(D, R)
            print(f"epilogue {name} ({out}): rel err {err:.3e}")
            assert err < 5e-6
    if f is not None and s is not None:     # both planes come from the same fp32 value
        assert (s - f).abs().max().item() <= 2.0 ** -20 * f.abs().max().item()


def _cross_k(L, xh, xl, wh, wl, Bn, T, d, head_major):
    """K head-major [Bn][H][T][64] of xa [Bn][T][d] and W_k [d][d]: one full-width GEMM with head_cols = 64, or one
    per-head batched GEMM of N = 64"""
    H = d // 64
    out_hi = torch.full((Bn, H, T, 64), float("nan"), dtype=torch.float16, device="cuda")
    out_lo = torch.full_like(out_hi, float("nan"))
    a = L.Operand(L.ptr(xh), L.ptr(xl), T, d, d, 0, T * d)
    ep = L.Epilogue()
    ep.out_hi, ep.out_lo, ep.ld_out = L.ptr(out_hi), L.ptr(out_lo), 64
    ep.out_h_stride, ep.out_b_stride, ep.alpha = T * 64, H * T * 64, 1.0
    if head_major:
        ep.head_cols = 64
        b = L.Operand(L.ptr(wh), L.ptr(wl), d, d, d, 0, 0)
        L.check(L.lib().stb_gemm(ctypes.byref(a), ctypes.byref(b), Bn, 1, ctypes.byref(ep), L.stream_ptr()))
    else:
        b = L.Operand(L.ptr(wh), L.ptr(wl), 64, d, d, 64 * d, 0)
        L.check(L.lib().stb_gemm(ctypes.byref(a), ctypes.byref(b), Bn, H, ctypes.byref(ep), L.stream_ptr()))
    torch.cuda.synchronize()
    return out_hi, out_lo


@pytest.mark.parametrize("Bn,T,d", [(3, 300, 384), (2, 1500, 1280)])
def test_head_major_columns(L, Bn, T, d):
    g = torch.Generator(device="cuda").manual_seed(d)
    x = torch.randn(Bn, T, d, device="cuda", generator=g)
    w = torch.randn(d, d, device="cuda", generator=g) * 0.05
    xh, xl = _split(x)
    wh, wl = _split(w)
    hm = _cross_k(L, xh, xl, wh, wl, Bn, T, d, True)
    ph = _cross_k(L, xh, xl, wh, wl, Bn, T, d, False)
    assert torch.equal(hm[0], ph[0]) and torch.equal(hm[1], ph[1]), "head-major differs from the per-head GEMMs"
    D = (hm[0].double() + hm[1].double()).cpu()
    R = (x.double().cpu() @ w.double().cpu().T).view(Bn, T, d // 64, 64).permute(0, 2, 1, 3)
    err = _rel(D, R)
    print(f"head-major cross K {Bn}x{T}x{d}: rel err {err:.3e}")
    assert err < max(5e-6, 4e-7 * d ** 0.5)       # grows ~sqrt(K), as in test_gpu_kernels


def test_head_cols_argument_checks(L):
    x = torch.zeros(128, 128, dtype=torch.float16, device="cuda")
    a = L.Operand(L.ptr(x), None, 128, 128, 128, 0, 0)
    ep = L.Epilogue()
    ep.out_hi, ep.ld_out, ep.alpha, ep.head_cols = L.ptr(x), 64, 1.0, 63
    assert L.lib().stb_gemm(ctypes.byref(a), ctypes.byref(a), 1, 1, ctypes.byref(ep), L.stream_ptr()) != 0
    ep.head_cols, ep.transposed = 64, 1
    assert L.lib().stb_gemm(ctypes.byref(a), ctypes.byref(a), 1, 1, ctypes.byref(ep), L.stream_ptr()) != 0


def test_two_calls_bitwise_equal(L):
    M, N, K = 128 * 5 * _sms() + 9, 1280, 1280
    A, B = _inputs(M, N, K, 3)
    g = torch.Generator(device="cuda").manual_seed(4)
    bias = torch.randn(N, device="cuda", generator=g)
    f1, s1 = _run(L, A, B, bias=bias, act=1, out="both")
    f2, s2 = _run(L, A, B, bias=bias, act=1, out="both")
    assert torch.equal(f1, f2) and torch.equal(s1, s2)
