"""Exact restatement of the tensor-core split-bf16 scheme (csrc/gemm_tc.cuh) for operands on which every kernel must give
known bits.

Operands are dyadic: the values of A are multiples of 2^-qa, those of B of 2^-qb, the bias of 2^-(qa+qb).  If for every
output (sum over k and over the kept plane products of |a_p b_q|) + |bias| is below 2^22 quanta of 2^-(qa+qb), every
partial sum in any order is an fp32 value of at most 22 significant bits, so every fp32 add, every truncated wgmma
result and every unbias_rz (r plus half an ulp of r is a tie that rounds back to r, whose last mantissa bit is zero) is
exact.  The kernel's output is then the fp64 sum of exactly the products the scheme keeps (`scheme_ref`), bit for bit.

The planes are the RN-even residual split p0 = bf16(x), p1 = bf16(x - p0), ... that split4 and tc_prep_weights_body
compute.  `bf16_rn` restates cvt.rn.bf16.f32 on the bit pattern, so that subnormal values round as on the device
whatever vector instructions the host's torch uses for its own bf16 conversion.  Works on CPU and CUDA tensors."""
import math

import torch

KEPT = {2: [(0, 0), (0, 1), (1, 0)],                              # hi*hi, hi*lo, lo*hi
        3: [(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)]}      # + mid*mid, hi*lo, lo*hi: every product of weight >= 2^-16
BUDGET_BITS = 22
NT = {2: 256, 3: 128}                                             # nt_of: rows of a weight-image tile


# ---- planes -----------------------------------------------------------------------------------------------------------
def bf16_rn(x):
    """fp32 -> bf16 (round to nearest even) -> fp32, on the bits; finite inputs"""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return torch.where(r >= 2 ** 31, r - 2 ** 32, r).to(torch.int32).view(torch.float32)


def planes(x, np_):
    """[p0, p1, ...]: p0 = bf16(x), p_i = bf16(what the planes before it left), each an fp32 tensor"""
    r = x.to(torch.float32)
    out = []
    for _ in range(np_):
        p = bf16_rn(r)
        out.append(p)
        r = r - p
    return out


def plane_bits(x, np_):
    """the planes as the uint16 bits the device stores, in an int16 tensor [np_, *x.shape]"""
    return torch.stack([(p.view(torch.int32) >> 16).to(torch.int16) for p in planes(x, np_)])


def residual(x, np_):
    return x.to(torch.float32) - sum(planes(x, np_))


# ---- references -------------------------------------------------------------------------------------------------------
def scheme_ref(A, B, bias, np_):
    """fp64 sum of exactly the kept plane products: A [M, K], B [N, K] (B(n, k)), bias [N] or None -> [M, N]"""
    pa, pb = planes(A, np_), planes(B, np_)
    y = sum(pa[p].double() @ pb[q].double().t() for p, q in KEPT[np_])
    return y if bias is None else y + bias.double()


def full_ref(A, B, bias):
    y = A.double() @ B.double().t()
    return y if bias is None else y + bias.double()


def abs_kept(A, B, bias, np_):
    """per output: the sum over k and the kept products of |a_p b_q|, plus |bias|"""
    pa, pb = planes(A, np_), planes(B, np_)
    y = sum(pa[p].double().abs() @ pb[q].double().abs().t() for p, q in KEPT[np_])
    return y if bias is None else y + bias.double().abs()


def quantum_exp(x):
    """the largest q such that every value of x is a multiple of 2^-q (0 for an all-zero tensor)"""
    v = x.double().flatten()
    v = v[v != 0]
    if v.numel() == 0:
        return 0
    m, e = torch.frexp(v)                                           # v = m 2^e, 0.5 <= |m| < 1
    mi = (m.abs() * 2.0 ** 53).to(torch.int64)
    tz = (mi & -mi).double().log2().round().to(torch.int64)         # trailing zero bits of the 53-bit mantissa
    return int(-(e.to(torch.int64) - 53 + tz).min())


def budget_bits(A, B, bias, np_):
    """log2 of the largest per-output sum of kept |products| (+ |bias|) in quanta of 2^-(qa + qb)"""
    q = quantum_exp(A) + quantum_exp(B)
    if bias is not None:
        assert quantum_exp(bias) <= q, "the bias must be a multiple of 2^-(qa + qb)"
    s = float(abs_kept(A, B, bias, np_).max())
    return math.log2(s) + q if s > 0 else -math.inf


def lo_fraction(x, np_, plane=1):
    """the fraction of the nonzero elements of x whose plane `plane` is nonzero"""
    nz = x != 0
    return float((planes(x, np_)[plane][nz] != 0).double().mean()) if bool(nz.any()) else 0.0


# ---- operand families -------------------------------------------------------------------------------------------------
# (name, description).  "a" / "b" suffixes say which operand carries the extra planes; the other is hi-only (integers).
FAMILIES = {
    "F0": "small integers on both sides, dense: any misplaced row, column, K slice, tile, split or stale stage changes bits",
    "F1a": "A with two nonzero planes (i + j/256, j odd), B hi-only: lo*hi (2 planes) / mid*hi (3 planes) must be kept",
    "F1b": "A hi-only, B with two nonzero planes: hi*lo / hi*mid must be kept",
    "F2a": "A with three nonzero planes (20-bit values), B hi-only and sparse: lo*hi (3 planes) must be kept",
    "F2b": "A hi-only and sparse, B with three nonzero planes: hi*lo (3 planes) must be kept",
    "F3": "both with a nonzero second plane, B sparse: lo*lo (2 planes, dropped) or mid*mid (3 planes, kept) is not zero",
}
MIN_FRACTION = 0.3      # of the nonzero elements of a multi-plane operand whose last exercised plane is nonzero


def _ints(shape, lim, g, device):
    return torch.randint(-lim, lim + 1, shape, generator=g, device=device).to(torch.float32)


def _two_plane(shape, g, device):
    """i + j / 256, i in [-3, 3], j odd in [-127, 127]: at most 10 significant bits, exactly hi + lo; lo != 0 unless i = 0"""
    j = torch.randint(-64, 64, shape, generator=g, device=device) * 2 + 1
    return _ints(shape, 3, g, device) + j.to(torch.float32) / 256


def _three_plane(shape, g, device):
    """m 2^-21 with 2^19 <= |m| < 2^20: 20 significant bits in (-0.5, 0.5), exactly hi + mid + lo"""
    m = torch.randint(2 ** 19, 2 ** 20, shape, generator=g, device=device)
    s = torch.randint(0, 2, shape, generator=g, device=device) * 2 - 1
    return ((m * s).double() * 2.0 ** -21).to(torch.float32)


def sparse_rows(rows, K, nnz, g, device, lim=1):
    """[rows, K] integers in [-lim, lim] \\ {0} at (at most) nnz random columns per row, zeros elsewhere"""
    out = torch.zeros(rows, K, device=device)
    cols = torch.randint(0, K, (rows, nnz), generator=g, device=device)
    v = torch.randint(1, lim + 1, (rows, nnz), generator=g, device=device) * (torch.randint(0, 2, (rows, nnz), generator=g, device=device) * 2 - 1)
    out.scatter_(1, cols, v.to(torch.float32))
    return out


def family(name, M, N, K, np_, seed, device="cpu", bias=True, nnz=3, sparse=None):
    """(A [M, K], B [N, K], bias [N] or None) of a family, checked against its budget and plane occupancy: operands that
    break either are refused (AssertionError).  Sparse families keep nnz nonzeros (at most) per row of B, so that each
    output is a sum of at most nnz products; F0 / F1 are dense unless `sparse` is set (weight gradients over many
    points: the budget grows with the number of products)."""
    assert name in FAMILIES, name
    g = torch.Generator(device=device).manual_seed(seed)
    mask = lambda: sparse_rows(N, K, nnz, g, device) != 0          # noqa: E731
    if name == "F0":
        A, B, qbias = _ints((M, K), 3, g, device), _ints((N, K), 3, g, device), 0
        B = B * mask() if sparse else B
    elif name == "F1a":
        A, B, qbias = _two_plane((M, K), g, device), _ints((N, K), 3, g, device), 8
        B = B * mask() if sparse else B
    elif name == "F1b":
        A, B, qbias = _ints((M, K), 3, g, device), _two_plane((N, K), g, device), 8
        B = B * mask() if sparse else B
    elif name == "F2a":
        assert np_ == 3, "F2 exercises the third plane"
        A, B, qbias = _three_plane((M, K), g, device), sparse_rows(N, K, nnz, g, device), 21
    elif name == "F2b":
        assert np_ == 3, "F2 exercises the third plane"
        A, B, qbias = _ints((M, K), 1, g, device), _three_plane((N, K), g, device) * mask(), 21
    else:
        A, B, qbias = _two_plane((M, K), g, device), _two_plane((N, K), g, device) * mask(), 16
    b = None
    if bias:                                                       # |bias| < 2^min(19 - q, 6): 1/8 of the budget at most
        lim = 2 ** (min(BUDGET_BITS - 3 - qbias, 6) + qbias)
        b = (torch.randint(-lim + 1, lim, (N,), generator=g, device=device).double() * 2.0 ** -qbias).to(torch.float32)
    check_family(name, A, B, b, np_)
    return A, B, b


def check_family(name, A, B, bias, np_):
    bits = budget_bits(A, B, bias, np_)
    assert bits < BUDGET_BITS, (name, bits)
    need = {"F1a": [(A, 1)], "F1b": [(B, 1)], "F2a": [(A, 2)], "F2b": [(B, 2)], "F3": [(A, 1), (B, 1)]}.get(name, [])
    for x, plane in need:
        frac = lo_fraction(x, np_, plane)
        assert frac >= MIN_FRACTION, (name, plane, frac)
        assert bool((residual(x, np_)[x != 0] == 0).all()), (name, "not exact in %d planes" % np_)
    return bits


# ---- the kernels' summation orders, emulated in fp32 ------------------------------------------------------------------
def rz32(x):
    """fp64 -> fp32 rounded toward zero: a wgmma result"""
    f = x.to(torch.float32)
    over = f.double().abs() > x.abs()
    return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f)


def unbias_rz(r):
    """r + half an ulp of r with the sign of r (its exponent bits times 2^-24), one rounding: csrc/gemm_tc.cuh"""
    e = (r.view(torch.int32) & -8388608).view(torch.float32)       # 0xff800000: sign and exponent
    return (r.double() + e.double() * 2.0 ** -24).to(torch.float32)


def _step(pa, pb, p, q, k0, k1):
    return pa[p][:, k0:k1].double() @ pb[q][:, k0:k1].double().t()


def emulate_w2(A, B, bias):
    """gemm_w_kernel: per 16-wide K step lo*hi, hi*lo, hi*hi, each wgmma truncating into one running accumulator"""
    pa, pb = planes(A, 2), planes(B, 2)
    acc = torch.zeros(A.shape[0], B.shape[0], dtype=torch.float32, device=A.device)
    for k0 in range(0, A.shape[1], 16):
        for p, q in ((1, 0), (0, 1), (0, 0)):
            acc = rz32(acc.double() + _step(pa, pb, p, q, k0, k0 + 16))
    return acc if bias is None else acc + bias


def emulate_w3(A, B, bias):
    """gemm_w3_tma_kernel: per 64-wide slice the five corrections into a zeroed accumulator, then each 16-wide hi*hi
    step into fresh registers; tot += corrections, tot += unbias_rz(hh0) .. unbias_rz(hh3) in fp32"""
    pa, pb = planes(A, 3), planes(B, 3)
    tot = torch.zeros(A.shape[0], B.shape[0], dtype=torch.float32, device=A.device)
    for s0 in range(0, A.shape[1], 64):
        corr = torch.zeros_like(tot)
        for k0 in range(s0, s0 + 64, 16):
            for p, q in ((2, 0), (0, 2), (1, 1), (1, 0), (0, 1)):
                corr = rz32(corr.double() + _step(pa, pb, p, q, k0, k0 + 16))
        tot = tot + corr
        for k0 in range(s0, s0 + 64, 16):
            tot = tot + unbias_rz(rz32(_step(pa, pb, 0, 0, k0, k0 + 16)))
    return tot if bias is None else tot + bias


def emulate_tn(A, B, C0, k_chunk):
    """gemm_tn_kernel + splitk_reduce_kernel: C0 + the split partials (each over k_chunk points in 16-point steps of
    lo*hi, hi*lo, hi*hi) summed in split order; one split adds its partial to C0 directly"""
    K = A.shape[1]
    parts = [emulate_w2(A[:, k0:k0 + k_chunk], B[:, k0:k0 + k_chunk], None) for k0 in range(0, K, k_chunk)]
    if len(parts) == 1:
        return C0 + parts[0]
    x = torch.zeros_like(parts[0])
    for part in parts:
        x = x + part
    return C0 + x


# ---- the weight image of nudf_tc_prepare_weights ----------------------------------------------------------------------
def pad16(n):
    return (n + 15) // 16 * 16


def pad64(k):
    return (k + 63) // 64 * 64


def tile_rows(N, t, np_):
    return pad16(min(N - NT[np_] * t, NT[np_]))


def image_elems(N, K, np_):
    return sum(pad64(K) // 64 * np_ * tile_rows(N, t, np_) * 64 for t in range((N + NT[np_] - 1) // NT[np_]))


def sw128(row, k):
    """byte offset of (row, k) in a [rows x 64] bf16 K-major SWIZZLE_128B tile"""
    return (row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ (row & 7)) & 7) << 4) + ((k & 7) << 1)


def weight_image(W, N, K, transposed, np_):
    """the uint16 image (as int16) of B(n, k) = W[n, k] (transposed = 0) or W[k, n] (1): n-tiles of nt_of(np_) rows, the
    last padded to 16, k-slices of 64 (K padded to pad64(K)), order [n-tile][k-slice][plane][rows x 128 B SW128], zeros
    in the padding"""
    Bm = (W[:K, :N].t() if transposed else W[:N, :K]).to(torch.float32)
    Kp, dev = pad64(K), W.device
    img = torch.zeros(image_elems(N, K, np_), dtype=torch.int16, device=dev)
    off = 0
    for t in range((N + NT[np_] - 1) // NT[np_]):
        rows = tile_rows(N, t, np_)
        blk = torch.zeros(rows, Kp, dtype=torch.float32, device=dev)
        n0 = t * NT[np_]
        blk[:min(N - n0, rows), :K] = Bm[n0:n0 + rows]
        bits = plane_bits(blk, np_)                                  # [np, rows, Kp]
        r = torch.arange(rows, device=dev)[:, None]
        k = torch.arange(64, device=dev)[None, :]
        sw = sw128(r, k) >> 1                                        # [rows, 64] in uint16 units
        s = torch.arange(Kp // 64, device=dev)[:, None, None, None]
        p = torch.arange(np_, device=dev)[None, :, None, None]
        idx = off + (s * np_ + p) * rows * 64 + sw[None, None]      # [S, np, rows, 64]
        val = bits.reshape(np_, rows, Kp // 64, 64).permute(2, 0, 1, 3)
        img[idx.flatten()] = val.flatten()
        off += Kp // 64 * np_ * rows * 64
    assert off == img.numel()
    return img


# ---- the split over the points of gemm_tn (tn_k_chunk in csrc/gemm_tc.cuh) ------------------------------------------
TN_WAVE_CTAS, TN_MIN_POINTS, SPLIT_WS_FLOATS = 132, 512, 8 << 20


def tn_k_chunk(M, N, K):
    cd = lambda a, b: (a + b - 1) // b                               # noqa: E731
    tiles = cd(M, 128) * cd(N, 128)
    splits = min(TN_WAVE_CTAS // tiles, cd(K, TN_MIN_POINTS))
    want, per = max(splits, 1), M * N + M
    cap = SPLIT_WS_FLOATS // per
    splits = want if want < cap else max(cap, 1)
    return cd(cd(K, splits), 64) * 64
