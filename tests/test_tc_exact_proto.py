"""The exact-arithmetic oracle of the tensor-core kernels (tests/proto/tc_exact.py) on the host: every operand family
meets its budget and exercises the planes it is there for, the kernels' summation orders emulated in fp32 (truncated
wgmma results, unbias_rz, split-K partials) give exactly scheme_ref on them, and the reference can tell a kept product
from a dropped one.  tests/test_gpu_tc_exact.py then holds the kernels to scheme_ref bit for bit."""
import pytest
import torch

from tests.proto import tc_exact as T

CASES = [("F0", 2), ("F0", 3), ("F1a", 2), ("F1a", 3), ("F1b", 2), ("F1b", 3), ("F2a", 3), ("F2b", 3), ("F3", 2), ("F3", 3)]
SHAPES = [(16, 16, 16), (77, 129, 259), (33, 40, 64), (20, 24, 39)]   # (M, N, K)


def test_bf16_rn_is_round_to_nearest_even():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(100000, generator=g) * 2.0 ** torch.randint(-60, 60, (100000,), generator=g).float()
    assert torch.equal(T.bf16_rn(x), x.to(torch.bfloat16).float())
    # ties go to the even neighbour, carries reach the exponent, subnormals round on their own grid
    one = torch.tensor([1.0])
    tie_down = one + 2.0 ** -8                                        # halfway between 1 and 1 + 2^-7, even: 1
    tie_up = one + 3 * 2.0 ** -8                                      # halfway between 1 + 2^-7 and 1 + 2^-6, even: 1 + 2^-6
    carry = torch.tensor([2.0 - 2.0 ** -9])
    sub = torch.tensor([2.0 ** -130 + 2.0 ** -140, -(2.0 ** -140)], dtype=torch.float64).float()
    assert float(T.bf16_rn(tie_down)) == 1.0
    assert float(T.bf16_rn(tie_up)) == 1.0 + 2.0 ** -6
    assert float(T.bf16_rn(carry)) == 2.0
    assert T.bf16_rn(sub).tolist() == [2.0 ** -130, -0.0]


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("name,np_", CASES)
def test_family_meets_budget_and_occupancy(name, np_, M, N, K):
    A, B, bias = T.family(name, M, N, K, np_, seed=M + N + K)
    assert T.check_family(name, A, B, bias, np_) < T.BUDGET_BITS
    for x in (A, B):
        assert bool((T.residual(x, np_) == 0).all())                 # every operand is exactly the sum of its planes


def test_family_refuses_operands_over_budget():
    with pytest.raises(AssertionError):
        T.family("F1a", 64, 64, 16384, 2, seed=1)                    # dense: 16384 products of up to 3.5 x 3, 2^-8 quanta
    T.family("F1a", 64, 64, 16384, 2, seed=1, sparse=True)
    A, B, b = T.family("F3", 16, 16, 64, 2, seed=1)
    with pytest.raises(AssertionError):
        T.check_family("F3", A, torch.ones_like(B) / 3, b, 2)         # 1/3 is neither dyadic enough nor two planes


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("name,np_", CASES)
def test_summation_orders_are_exact(name, np_, M, N, K):
    A, B, bias = T.family(name, M, N, K, np_, seed=3 * M + N + K)
    ref = T.scheme_ref(A, B, bias, np_)
    emulate = T.emulate_w2 if np_ == 2 else T.emulate_w3
    Kp = T.pad64(K)                                                   # the kernels see zeros past K
    Ap = torch.nn.functional.pad(A, (0, Kp - K))
    Bp = torch.nn.functional.pad(B, (0, Kp - K))
    assert torch.equal(emulate(Ap, Bp, bias).double(), ref)
    if np_ == 2:                                                      # the same family as a weight gradient
        C0 = (torch.randint(-64, 64, (M, N)).double() * 2.0 ** -T.quantum_exp(A)).float()
        for k_chunk in (64, 128, Kp):
            assert torch.equal(T.emulate_tn(Ap, Bp, C0, k_chunk).double(), C0.double() + T.scheme_ref(A, B, None, 2))


def test_unbias_rz_is_exact_on_short_values_and_centres_truncation():
    g = torch.Generator().manual_seed(2)
    r = (torch.randint(-2 ** 22 + 1, 2 ** 22, (10000,), generator=g).double() * 2.0 ** -7).float()
    assert torch.equal(T.unbias_rz(r), r)                            # at most 22 significant bits: a tie back to r
    x = torch.randn(200000, generator=g, dtype=torch.float64) * 100
    t = T.rz32(x)
    assert bool((t.double().abs() <= x.abs()).all())
    rel = lambda y: ((y.double() - x) * x.sign() / x.abs()).mean().item() * 2 ** 24   # noqa: E731
    assert rel(t) < -0.3                                             # truncation: about -0.7 ulp(2^-24) on average
    assert abs(rel(T.unbias_rz(t))) < 0.05


@pytest.mark.parametrize("np_", [2, 3])
def test_f3_tells_kept_from_dropped_products(np_):
    A, B, bias = T.family("F3", 40, 48, 259, np_, seed=9)
    s, f = T.scheme_ref(A, B, bias, np_), T.full_ref(A, B, bias)
    pa, pb = T.planes(A, np_), T.planes(B, np_)
    if np_ == 2:
        assert not torch.equal(s, f)
        assert torch.equal(f - s, pa[1].double() @ pb[1].double().t())   # lo*lo, and nothing else, is dropped
        assert (s != f).double().mean().item() > 0.5
    else:
        assert torch.equal(s, f)
        mm = pa[1].double() @ pb[1].double().t()                          # mid*mid is kept and not zero
        assert (mm != 0).double().mean().item() > 0.5


@pytest.mark.parametrize("np_", [2, 3])
@pytest.mark.parametrize("transposed", [0, 1])
@pytest.mark.parametrize("N,K", [(16, 16), (40, 39), (129, 70), (257, 20)])
def test_weight_image_layout(N, K, transposed, np_):
    """weight_image against a per-element restatement of tc_prep_weights_body's index arithmetic"""
    g = torch.Generator().manual_seed(N + K)
    W = torch.randn((K, N) if transposed else (N, K), generator=g)
    img = T.weight_image(W, N, K, transposed, np_)
    assert img.numel() == T.image_elems(N, K, np_)
    Kp, nt = T.pad64(K), T.NT[np_]
    bits = T.plane_bits(W, np_).tolist()
    got = img.tolist()
    seen = [False] * len(got)
    off = 0
    for t in range((N + nt - 1) // nt):
        rows = T.tile_rows(N, t, np_)
        for nl in range(rows):
            n = t * nt + nl
            for k in range(Kp):
                for p in range(np_):
                    i = off + ((k // 64) * np_ + p) * rows * 64 + (T.sw128(nl, k % 64) >> 1)
                    want = 0 if n >= N or k >= K else (bits[p][k][n] if transposed else bits[p][n][k])
                    assert got[i] == want, (t, nl, k, p)
                    seen[i] = True
        off += Kp // 64 * np_ * rows * 64
    assert all(seen)
