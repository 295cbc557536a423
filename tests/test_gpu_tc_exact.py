"""The tensor-core kernels held to exact results (tests/proto/tc_exact.py): on dyadic operands within the 22-bit budget
every layer (gemm_w_kernel, gemm_w3_tma_kernel) and weight-gradient (gemm_tn_kernel + splitk_reduce_kernel) result is
the fp64 sum of exactly the plane products the scheme keeps, so the kernel must reproduce it bit for bit at every shape
its tiling, ring slots, persistent grid and split over the points branch on.  The weight image must be the host's plane
split bit for bit.  On general fp32 operands each output is held to a per-element bound derived from the scheme, and the
3-plane kernel's correction of the tensor core's truncation toward zero must hold."""
import math

import pytest
import torch

from tests.gpu_util import report
from tests.proto import tc_exact as T

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24                      # unit roundoff of fp32
NAN = float("nan")
SENTINEL = 7.0


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _lib():
    from neuraludf_b200 import _lib as L
    return L, L.lib()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _image(Bm, N, K, transposed, np_):
    """nudf_tc_prepare_weights of B(n, k) = Bm[n, k], from W = Bm (transposed 0) or W = Bm^T (1); the image buffer is
    pre-filled with a pattern no plane split produces here, so that an element left unwritten shows"""
    L, lib = _lib()
    W = Bm.t().contiguous() if transposed else Bm.contiguous()
    img = torch.full((lib.nudf_tc_image_elems(N, K, np_),), 0x5A5A, dtype=torch.int16, device=DEV)
    L.check(lib.nudf_tc_prepare_weights(L.ptr(W), W.stride(0), N, K, transposed, np_, L.ptr(img), L.stream_ptr()), "prep")
    return img, W


def _padded(X):
    """X [rows, width] in a buffer with a row stride of round_up(width, 4) + 4 floats, NaN in the padding columns"""
    rows, width = X.shape
    ld = (width + 3) // 4 * 4 + 4
    buf = torch.full((rows, ld), NAN, device=DEV)
    buf[:, :width] = X
    return buf


def _layer(A, img, np_, bias, N, act=0, engine=1, W=None):
    """Y = act(A B^T + bias) into a NaN-filled [M + 2, N + 5] buffer; checks that nothing outside [M, N] was written"""
    L, lib = _lib()
    M, K = A.shape
    X = _padded(A)
    Y = torch.full((M + 2, N + 5), NAN, device=DEV)
    if engine == 1:
        L.check(lib.nudf_dense_forward_tc(L.ptr(X), X.stride(0), L.ptr(img), np_, L.ptr(bias), L.ptr(Y), Y.stride(0), M, N,
                                          K, act, L.stream_ptr()), "dense_forward_tc")
    else:
        L.check(lib.nudf_dense_forward(L.ptr(X), X.stride(0), L.ptr(W), W.stride(0), L.ptr(bias), L.ptr(Y), Y.stride(0), M,
                                       N, K, act, L.stream_ptr()), "dense_forward")
    torch.cuda.synchronize()
    outside = torch.ones_like(Y, dtype=torch.bool)
    outside[:M, :N] = False
    assert bool(torch.isnan(Y[outside]).all()), "write outside [M, N]"
    return Y[:M, :N]


def _exact(ref):
    """scheme_ref as the fp32 tensor the kernel must produce (it is representable: the budget holds)"""
    y = ref.to(torch.float32)
    assert torch.equal(y.double(), ref)
    return y


def _first_diff(Y, ref, tag):
    bad = (Y != ref).nonzero()
    if bad.numel() == 0:
        return ""
    r, c = bad[0].tolist()
    return "%s: %d wrong elements, first (%d, %d): %r != %r" % (tag, bad.shape[0], r, c, float(Y[r, c]), float(ref[r, c]))


# ---- premise ----------------------------------------------------------------------------------------------------------
def test_premise_single_wgmma_window():
    """One 16-product wgmma step (a 2-plane layer with K = 16 on hi-only operands: the lo * hi and hi * lo steps add
    zeros) of row w: 2^w, fourteen ones, -2^w.  The exact sum 14 survives only if the tensor core keeps the ones next to
    2^w, i.e. if its accumulation window is wider than w bits.  The scheme's exactness needs every w < 22; the widths at
    which the ones are lost are reported (the measured window)."""
    ws = list(range(8, 40))
    A = torch.ones(len(ws), 16, device=DEV)
    for i, w in enumerate(ws):
        A[i, 0], A[i, 15] = 2.0 ** w, -(2.0 ** w)
    B = torch.ones(16, 16, device=DEV)
    img, _ = _image(B, 16, 16, 0, 2)
    Y = _layer(A, img, 2, None, 16)
    exact = (Y == 14).all(dim=1).tolist()
    window = next((w for w, ok in zip(ws, exact) if not ok), None)
    report("tc_exact.window", first_inexact_w=window, values=[float(v) for v in Y[:, 0].tolist()])
    assert all(ok for w, ok in zip(ws, exact) if w < T.BUDGET_BITS), Y[:, 0].tolist()


@pytest.mark.parametrize("name", ["F0", "F1a", "F1b"])
@pytest.mark.parametrize("np_", [2, 3])
def test_premise_small_exact(np_, name):
    """F0 and F1 at one tile: if these fail, the accumulation window is narrower than the families assume"""
    A, B, bias = T.family(name, 128, 128, 64, np_, seed=5, device=DEV)
    img, _ = _image(B, 128, 64, 0, np_)
    Y = _layer(A, img, np_, bias, 128)
    ref = _exact(T.scheme_ref(A, B, bias, np_))
    assert torch.equal(Y, ref), _first_diff(Y, ref, name)


# ---- layers, exact ----------------------------------------------------------------------------------------------------
def _tiles_m(tiles, N):
    """a row count whose 3-plane tile count (128 x 128 tiles) is `tiles`, ragged in its last row block where possible"""
    n_ct = (N + 127) // 128
    assert tiles % n_ct == 0
    return tiles // n_ct * 128 - 5


# (M, N, K): every N of the WN = 128 / 256 switch and image padding (217 -> 224, 257 -> 272), every K edge (one step,
# a ragged last slice, ring-slot reuse: 3 slots at WN = 256, 4 at WN = 128, 2 stages of the 3-plane kernel) and
# M from one row to a ragged 512th row block
LAYER_SHAPES = [(1, 16, 16), (77, 128, 39), (128, 129, 64), (129, 217, 256), (65499, 256, 259), (77, 257, 259),
                (129, 16, 259), (128, 256, 16), (1, 257, 64), (65499, 129, 39), (77, 217, 16), (1000, 257, 256)]


def _tile_shapes():
    """3-plane tile counts S - 1, S, S + 1, 2S + 1 and a large count that S does not divide, S = the device's SMs
    (the persistent grid is min(tiles, SMs) CTAs)"""
    S = _sms()
    return [(_tiles_m(S - 1, 128), 128, 259), (_tiles_m(S, 128), 128, 64), (_tiles_m(S + 1, 128), 128, 39),
           (_tiles_m(2 * S + 1, 128), 128, 256), (65499, 257, 259)]


def _check_layer(M, N, K, np_, transposed, name, seed):
    A, B, bias = T.family(name, M, N, K, np_, seed=seed, device=DEV)
    img, _ = _image(B, N, K, transposed, np_)
    Y = _layer(A, img, np_, bias, N)
    ref = _exact(T.scheme_ref(A, B, bias, np_))
    tag = "%s np%d t%d [%d,%d,%d]" % (name, np_, transposed, M, N, K)
    assert torch.equal(Y, ref), _first_diff(Y, ref, tag)
    if name == "F3" and np_ == 2:
        assert not torch.equal(Y.double(), T.full_ref(A, B, bias))    # lo * lo is dropped, and the test can tell


@pytest.mark.parametrize("transposed", [0, 1])
@pytest.mark.parametrize("np_", [2, 3])
@pytest.mark.parametrize("M,N,K", LAYER_SHAPES)
def test_layer_exact_f0(M, N, K, np_, transposed):
    _check_layer(M, N, K, np_, transposed, "F0", seed=M + 3 * N + 7 * K + transposed)


@pytest.mark.parametrize("case", range(5))
def test_layer3_exact_persistent_tiles(case):
    """the 3-plane kernel at tile counts around and above the persistent grid: cross-tile stage parity and landing
    quarters refilled with the next tile's rows"""
    M, N, K = _tile_shapes()[case]
    for name in ("F0", "F2a"):
        _check_layer(M, N, K, 3, case & 1, name, seed=11 * case + len(name))


@pytest.mark.parametrize("name", ["F1a", "F1b", "F3"])
@pytest.mark.parametrize("np_", [2, 3])
@pytest.mark.parametrize("M,N,K", [(65499, 257, 259), (129, 129, 39), (77, 217, 64)])
def test_layer_exact_planes(M, N, K, np_, name):
    """each kept cross-plane product reaches the output: lo * hi and hi * lo (2 planes), mid * hi, hi * mid, mid * mid
    (3 planes); F3 also shows that lo * lo is dropped from 2-plane layers"""
    _check_layer(M, N, K, np_, (M + K) & 1, name, seed=M + N + K + len(name))


@pytest.mark.parametrize("name", ["F2a", "F2b"])
@pytest.mark.parametrize("M,N,K", [(65499, 257, 259), (129, 129, 39), (1000, 16, 256)])
def test_layer3_exact_third_plane(M, N, K, name):
    """lo * hi and hi * lo of the 3-plane layers on 20-bit operands (three nonzero planes)"""
    _check_layer(M, N, K, 3, K & 1, name, seed=M + N + K + len(name))


# ---- activations ------------------------------------------------------------------------------------------------------
def _ulp(x):
    a = x.abs().to(torch.float32)
    return (torch.nextafter(a, torch.full_like(a, math.inf)) - a).double()


@pytest.mark.parametrize("act", [0, 1, 2, 3])
@pytest.mark.parametrize("M,N,K", [(1000, 217, 259), (77, 128, 39)])
def test_activations_exact_preactivation(M, N, K, act):
    """F0 operands with B and the bias scaled by 2^-6 (z in steps of 2^-6, mostly within a few units of 0): the
    pre-activation is exact on every engine, so the FFMA engine and both tensor-core kernels give the same bits, and
    those are within a few ulp of the fp64 activation of the exact z.  softplus (beta 100) uses MUFU exp / log: its
    documented absolute error is 4e-9 on top of the rounding."""
    A, B, bias = T.family("F0", M, N, K, 2, seed=M + N + act, device=DEV)
    B, bias = B * 2.0 ** -6, bias * 2.0 ** -6
    z = T.full_ref(A, B, bias)
    assert torch.equal(z, T.scheme_ref(A, B, bias, 3)) and torch.equal(z, T.scheme_ref(A, B, bias, 2))
    ys = {}
    for np_ in (2, 3):
        img, _ = _image(B, N, K, 0, np_)
        ys["tc%d" % np_] = _layer(A, img, np_, bias, N, act=act)
    ys["ffma"] = _layer(A, None, 0, bias, N, act=act, engine=0, W=B.contiguous())
    for k, y in ys.items():
        assert torch.equal(y, ys["ffma"]), _first_diff(y, ys["ffma"], k)
    y = ys["ffma"].double()
    if act == 0:
        assert torch.equal(y, z)
    elif act == 1:
        assert torch.equal(y, z.clamp_min(0))
    elif act == 2:
        ref = torch.where(100 * z > 20, z, torch.log1p(torch.exp(100 * z)) / 100)
        err = ((y - ref).abs() - 4 * _ulp(ref)).max().item()
        report("tc_exact.softplus[%d,%d,%d]" % (M, N, K), err_over_4ulp=err)
        assert err <= 8e-9, err
    else:
        ref = torch.sigmoid(z)
        ulps = ((y - ref).abs() / _ulp(ref)).max().item()
        report("tc_exact.sigmoid[%d,%d,%d]" % (M, N, K), max_ulp=ulps)
        assert ulps <= 4, ulps


# ---- weight gradients, exact ------------------------------------------------------------------------------------------
def _wgrad(dZ, X, n_out, n_in, P, ldw, C0, engine):
    """dW [n_out, ldw] = C0 in the first n_in columns, SENTINEL beyond, += dZ^T X"""
    L, lib = _lib()
    dW = torch.full((n_out, ldw), SENTINEL, device=DEV)
    dW[:, :n_in] = C0
    L.check(lib.nudf_wgrad(L.ptr(dZ), dZ.stride(0), L.ptr(X), X.stride(0), n_out, n_in, P, L.ptr(dW), ldw, engine,
                           L.stream_ptr()), "wgrad")
    torch.cuda.synchronize()
    assert bool((dW[:, n_in:] == SENTINEL).all()), "write beyond n_in"
    return dW[:, :n_in]


def _check_wgrad(P, n_out, n_in, ldw, name, seed):
    # contraction over the points: A = dZ^T [n_out, P], B = X^T [n_in, P]
    A, B, _ = T.family(name, n_out, n_in, P, 2, seed=seed, device=DEV, bias=False, sparse=name != "F0")
    q = T.quantum_exp(A) + T.quantum_exp(B)
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    C0 = (torch.randint(-64, 64, (n_out, n_in), generator=g, device=DEV).double() * 2.0 ** -q).to(torch.float32)
    assert math.log2(float((T.abs_kept(A, B, None, 2) + C0.double().abs()).max())) + q < T.BUDGET_BITS
    dZ, X = A.t().contiguous(), B.t().contiguous()
    want = {1: _exact(C0.double() + T.scheme_ref(A, B, None, 2)), 0: _exact(C0.double() + T.full_ref(A, B, None))}
    splits = -(-P // T.tn_k_chunk(n_out, n_in, P))
    for engine in (1, 0):
        got = _wgrad(dZ, X, n_out, n_in, P, ldw, C0, engine)
        tag = "%s e%d [P %d, %d x %d, ldw %d, %d splits]" % (name, engine, P, n_out, n_in, ldw, splits)
        assert torch.equal(got, want[engine]), _first_diff(got, want[engine], tag)


WGRAD_SHAPES = [(256, 256), (217, 39), (128, 40)]     # (n_out, n_in): n_in = 256 and 40 reach red.global.add.v4


@pytest.mark.parametrize("ldw_pad", [0, 3])
@pytest.mark.parametrize("n_out,n_in", WGRAD_SHAPES)
@pytest.mark.parametrize("P", [77, 511, 512, 1000, 65499, 131072])
def test_wgrad_exact_f0(P, n_out, n_in, ldw_pad):
    """one split (P <= 512 at 256 x 256), several, slices that cross a chunk end and points past P; both engines"""
    _check_wgrad(P, n_out, n_in, n_in + ldw_pad, "F0", seed=P + n_out + n_in + ldw_pad)


@pytest.mark.parametrize("name", ["F1a", "F1b", "F3"])
@pytest.mark.parametrize("n_out,n_in", WGRAD_SHAPES)
@pytest.mark.parametrize("P", [1000, 131072])
def test_wgrad_exact_planes(P, n_out, n_in, name):
    """lo * hi and hi * lo of gemm_tn_kernel (sparse over the points to stay in the budget); on F3 the tensor-core
    engine drops lo * lo and the FFMA engine does not"""
    _check_wgrad(P, n_out, n_in, n_in, name, seed=P + n_out + len(name))


# ---- weight image -----------------------------------------------------------------------------------------------------
def _image_values(N, K, seed):
    """values that exercise the split: normal values over a wide range, +-0, residuals that are subnormal or flush to
    zero in bf16, and values whose bf16 rounding carries into the exponent"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(N, K, generator=g, device=DEV, dtype=torch.float64) * 2.0 ** torch.randint(-30, 30, (N, K), generator=g, device=DEV)
    m = torch.randint(1, 2 ** 16, (N, K), generator=g, device=DEV).double()
    kinds = [torch.zeros_like(x), -torch.zeros_like(x),
             2.0 ** -118 * (1 + m * 2.0 ** -23),                      # residual below 2^-126: subnormal
             2.0 ** -126 * (1 + m * 2.0 ** -23),                      # residual in the bf16 subnormal range and below
             m * 2.0 ** -149,                                         # subnormal values
             (2 - 2.0 ** -9 + m * 2.0 ** -40) * 2.0 ** torch.randint(-20, 20, (N, K), generator=g, device=DEV),   # carry
             -(1 + 2.0 ** -8) * torch.ones_like(x)]                   # a tie to even
    pick = torch.randint(0, len(kinds) + 3, (N, K), generator=g, device=DEV)
    for i, v in enumerate(kinds):
        x = torch.where(pick == i, v, x)
    return x.to(torch.float32)


@pytest.mark.parametrize("np_", [2, 3])
@pytest.mark.parametrize("transposed", [0, 1])
@pytest.mark.parametrize("N,K", [(16, 259), (128, 16), (129, 39), (217, 64), (256, 256), (257, 259), (257, 39), (217, 259)])
def test_weight_image_matches_host(N, K, transposed, np_):
    Bm = _image_values(N, K, seed=N * 7 + K + transposed)
    img, W = _image(Bm, N, K, transposed, np_)
    want = T.weight_image(W, N, K, transposed, np_)
    assert torch.equal(img, want), "%d elements differ" % int((img != want).sum())


# ---- general fp32 operands: per-element bounds and bias ---------------------------------------------------------------
# e = (Y - ref64) / (sum_k |a_k| |b_k| + |bias|) per output, u = 2^-24.  Planes: |a - a0| <= 2^-8 |a| (bf16 keeps 8
# significant bits), each further residual another factor 2^-8, so |a_i| <= 2^-8i (1 + 2^-8) |a|.
# * Dropped products, 2 planes: a1 b1, a0 rb, ra b0 and smaller: <= (3 + 2^-6) 2^-16 |a b|, taken as 3.1 * 2^-16.
#   3 planes: a1 b2, a2 b1 (2^-24 each), (a0 + a1 + a2) rb and ra (b0 + b1 + b2): <= 4.1 * 2^-24 |a b|.
# * A wgmma result is truncated toward zero once, after an internal alignment that may lose at most one more ulp: at
#   most 2 ulp, <= 2^-22 of the sum of the magnitudes it adds (<= 1.02 |a b| summed over its products).
# * Each fp32 add (the 3-plane kernel's tot, the split-K sums, the bias) rounds once: <= u of its magnitudes.
# gemm_w_kernel: 12 wgmma per 64-wide slice on one accumulator; gemm_w3_tma_kernel: 20 correction wgmma per slice
# (magnitudes <= 3.1 * 2^-8), 4 hi * hi results (each over its own 16 products, shifted by half an ulp), 5 fp32 adds per
# slice; gemm_tn_kernel: 3 wgmma per 16 points of a split, then one add per split; FFMA: one rounding per fma.
def bound_w2(K):
    return 3.1 * 2.0 ** -16 + 12 * T.pad64(K) // 64 * 1.02 * 2.0 ** -22 + U


def bound_w3(K):
    ns = T.pad64(K) // 64
    return 4.1 * U + 1.02 * 2.0 ** -22 + 20 * ns * 3.1 * 2.0 ** -8 * 2.0 ** -22 + (5 * ns + 1) * 1.02 * U


def bound_tn(n_out, n_in, P):
    kc = T.tn_k_chunk(n_out, n_in, P)
    return 3.1 * 2.0 ** -16 + 3 * (kc // 16) * 1.02 * 2.0 ** -22 + (-(-P // kc) + 1) * 1.02 * U


def bound_ffma_layer(K):
    return (K + 1) * 1.01 * U


def bound_ffma_wgrad(n_out, n_in, P):
    splits = min(-(-P // 2048), max(T.SPLIT_WS_FLOATS // (n_out * n_in), 1))
    kc = -(-(-(-P // splits)) // 8) * 8
    return (kc + splits + 1) * 1.01 * U


# rms(e), the largest measured at these shapes on an H100 80GB HBM3 (132 SMs, 700 W) times a margin of 2: gemm_w_kernel
# 9.3e-7 (K = 39), gemm_w3_tma_kernel 6.7e-8 (positive operands), gemm_tn_kernel 1.66e-6 (positive operands), FFMA 2.9e-8
RMS_BOUND = {"w2": 2e-6, "w3": 1.4e-7, "tn": 3.4e-6, "ffma": 6e-8}
# mean(e sign(ref)) / rms(e) of the 3-plane kernel on positive operands over 2^20 outputs: measured +0.213 with unbias_rz
# and -0.198 without it (the same H100).  The half ulp moves every truncated hi * hi result to the middle of its interval,
# but it also moves every exact one with an odd last bit up a whole ulp (a tie rounds to even), so the correction
# overshoots on operands whose 16-product sums are often exact.  The bounds hold the truncation toward zero corrected
# (t > -0.1) and the overshoot no larger than measured (t < 0.35).
BIAS_T_W3 = (-0.1, 0.35)


def _stats(tag, Y, ref, den, bound, kind):
    e = (Y.double() - ref) / den
    mx, rms = e.abs().max().item(), e.pow(2).mean().sqrt().item()
    t = ((e * ref.sign()).mean() / max(rms, 1e-300)).item()
    report("tc_exact.%s" % tag, max_e=mx, bound=bound, rms_e=rms, bias_t=t, n=e.numel())
    assert torch.isfinite(e).all(), tag
    assert mx <= bound, (tag, mx, bound)
    if RMS_BOUND[kind] is not None:
        assert rms <= RMS_BOUND[kind], (tag, rms)
    return t


def _general(M, N, K, seed, positive=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    if positive:
        return (torch.rand(M, K, generator=g, device=DEV), torch.rand(N, K, generator=g, device=DEV), None)
    return (torch.randn(M, K, generator=g, device=DEV), torch.randn(N, K, generator=g, device=DEV) / K ** 0.5,
            torch.randn(N, generator=g, device=DEV))


@pytest.mark.parametrize("M,N,K", [(65499, 257, 259), (-1, 128, 256), (1000, 217, 39)])
def test_layers_per_element_bound(M, N, K):
    if M < 0:
        M = _tiles_m(2 * _sms() + 1, N)
    A, B, bias = _general(M, N, K, seed=M + N + K)
    ref = T.full_ref(A, B, bias)
    den = A.double().abs() @ B.double().abs().t() + bias.double().abs()
    for np_ in (2, 3):
        img, _ = _image(B, N, K, 0, np_)
        Y = _layer(A, img, np_, bias, N)
        _stats("w%d[%d,%d,%d]" % (np_, M, N, K), Y, ref, den, bound_w2(K) if np_ == 2 else bound_w3(K), "w%d" % np_)
    Y = _layer(A, None, 0, bias, N, engine=0, W=B.contiguous())
    _stats("ffma[%d,%d,%d]" % (M, N, K), Y, ref, den, bound_ffma_layer(K), "ffma")


@pytest.mark.parametrize("P,n_out,n_in", [(65499, 256, 256), (131072, 128, 40), (1000, 217, 39)])
def test_wgrad_per_element_bound(P, n_out, n_in):
    A, B, _ = _general(n_out, n_in, P, seed=P + n_out)
    ref = T.full_ref(A, B, None)
    den = A.double().abs() @ B.double().abs().t()
    dZ, X = A.t().contiguous(), B.t().contiguous()
    Y = _wgrad(dZ, X, n_out, n_in, P, n_in, torch.zeros(n_out, n_in, device=DEV), 1)
    _stats("tn[%d,%d,%d]" % (P, n_out, n_in), Y, ref, den, bound_tn(n_out, n_in, P), "tn")
    Y = _wgrad(dZ, X, n_out, n_in, P, n_in, torch.zeros(n_out, n_in, device=DEV), 0)
    _stats("ffma_wgrad[%d,%d,%d]" % (P, n_out, n_in), Y, ref, den, bound_ffma_wgrad(n_out, n_in, P), "ffma")


def test_layer3_truncation_is_corrected():
    """Positive operands, so that every hi * hi result has the sign of the output: a truncation left uncorrected moves
    every output toward zero.  The 3-plane kernel's unbias_rz must undo that drift (BIAS_T_W3); the 2-plane kernel and
    gemm_tn_kernel make no claim about their bias and are reported only."""
    M, N, K = 8192, 128, 256
    A, B, _ = _general(M, N, K, seed=1, positive=True)
    ref = T.full_ref(A, B, None)
    den = A.double() @ B.double().t()
    t = {}
    for np_ in (3, 2):
        img, _ = _image(B, N, K, 0, np_)
        Y = _layer(A, img, np_, None, N)
        t[np_] = _stats("bias.w%d" % np_, Y, ref, den, bound_w2(K) if np_ == 2 else bound_w3(K), "w%d" % np_)
    P, n_out, n_in = 65536, 128, 128
    A, B, _ = _general(n_out, n_in, P, seed=2, positive=True)
    ref = T.full_ref(A, B, None)
    Y = _wgrad(A.t().contiguous(), B.t().contiguous(), n_out, n_in, P, n_in, torch.zeros(n_out, n_in, device=DEV), 1)
    t["tn"] = _stats("bias.tn", Y, ref, ref, bound_tn(n_out, n_in, P), "tn")
    report("tc_exact.bias", t_w3=t[3], t_w2=t[2], t_tn=t["tn"])
    assert BIAS_T_W3[0] < t[3] < BIAS_T_W3[1], t
