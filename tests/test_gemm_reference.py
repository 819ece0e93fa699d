"""CPU checks of the float64 GEMM / convolution statements in oracle/gemm64.py: every epilogue branch, batched and
broadcast strides, the relative-position skew and the accumulate form against the fp32 oracle/ops_ref.gemm; the nine-tap
convolution sums against torch's float64 conv2d / conv_transpose2d / autograd weight gradient."""
import pytest
import torch
import torch.nn.functional as F

from oracle import gemm64 as G
from oracle import ops_ref as R

BF = torch.bfloat16


def _bf(*shape, seed, scale=1.0, nonneg=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(*shape, generator=g) if nonneg else torch.randn(*shape, generator=g)
    return (x * scale).to(BF)


def _check(res, ref, what, rtol=2e-5):
    """ops_ref's fp32 result lies within a few fp32 roundings of the magnitude around the float64 value."""
    c = res.c.reshape(ref.shape)
    mag = res.mag.reshape(ref.shape)
    err = (ref.double() - c).abs()
    assert (err <= rtol * mag + 1e-30).all(), "%s: max err/mag %.3e" % (what, (err / mag.clamp_min(1e-30)).max())
    assert (c.abs() <= mag * (1 + 1e-12)).all(), "%s: magnitude below |value|" % what


def _epi_case(act, drop_mode, alpha, resid):
    M, N, K = 37, 45, 70
    A = _bf(M, K, seed=1)
    B = _bf(N, 72, seed=2)[:, :K]  # padded row stride
    bias = _bf(N, seed=3)
    kw = dict(bias=bias, act=act, alpha=alpha, drop_p=0.3 if drop_mode else 0.0, drop_mode=drop_mode, seed=77)
    if act in (G.ACT_RELU_BWD, G.ACT_SILU_BWD):
        aux = _bf(M, 48, seed=4)
        aux[::3, ::4] = 0  # ReLU' is strict at aux == 0
        kw.update(aux=aux, ld_aux=48)
    if resid == "bf16":
        kw.update(R=_bf(M, 56, seed=5), ldr=56, beta=-0.75)
    elif resid == "fp32":
        kw.update(R=torch.randn(M, N, generator=torch.Generator().manual_seed(6)), ldr=N, beta=1.5)
    return M, N, K, A, B, kw


@pytest.mark.parametrize("act", [G.ACT_NONE, G.ACT_RELU, G.ACT_SILU, G.ACT_RELU_BWD, G.ACT_SILU_BWD])
@pytest.mark.parametrize("drop_mode", [0, 1, 2])
@pytest.mark.parametrize("alpha,resid", [(1.0, None), (-0.375, "bf16"), (2.5, "fp32")])
def test_gemm64_epilogue_matches_ops_ref(act, drop_mode, alpha, resid):
    M, N, K, A, B, kw = _epi_case(act, drop_mode, alpha, resid)
    c2 = torch.empty(M, N, dtype=BF)
    ref = torch.empty(M, N)
    R.gemm(A, B, ref, M, N, K, K, 72, N, C2=c2, **kw)
    res = G.gemm(A, B, ref, M, N, K, K, 72, N, C2=c2, **kw)
    _check(res, ref, "epilogue")
    # the side output is bf16(acc + bias): within one bf16 rounding of the float64 pre-activation
    assert ((c2.double() - res.c2[0, 0]).abs() <= 2.0 ** -8 * res.c2[0, 0].abs() + 2e-5 * res.mag2[0, 0]).all()
    if act in (G.ACT_SILU, G.ACT_SILU_BWD):
        assert (res.apx > 0).any()
    else:
        assert not res.apx.any()


def test_gemm64_relu_bwd_is_strict_at_zero():
    M, N, K, A, B, kw = _epi_case(G.ACT_RELU_BWD, 0, 1.0, None)
    res = G.gemm(A, B, None, M, N, K, K, 72, N, **kw)
    u = kw["aux"][:, :N]
    assert (u == 0).any() and not res.c[0, 0][u == 0].any() and not res.mag[0, 0][u <= 0].any()


def test_gemm64_nonnegative_magnitude_is_value():
    A, B = _bf(50, 90, seed=8, nonneg=True), _bf(30, 90, seed=9, nonneg=True)
    res = G.gemm(A, B, None, 50, 30, 90, 90, 90, 30)
    assert torch.equal(res.c, res.mag)
    assert torch.equal(res.c[0, 0], A.double() @ B.double().t())


@pytest.mark.parametrize("ak,bk", [(True, True), (True, False), (False, True), (False, False)])
def test_gemm64_batched_broadcast_majors(ak, bk):
    nb1, nb2, M, N, K = 3, 2, 20, 24, 40
    a = _bf(nb2, nb1, M, K, seed=10)
    b = _bf(nb1, N, K, seed=11)  # broadcast along nb2
    A = a.contiguous() if ak else a.transpose(-1, -2).contiguous()
    Bm = b.contiguous() if bk else b.transpose(-1, -2).contiguous()
    lda, ldb = (K if ak else M), (K if bk else N)
    ldc = 32
    C = torch.zeros(nb2, nb1, M, ldc)
    kw = dict(a_kmajor=ak, b_kmajor=bk, nb1=nb1, nb2=nb2, sA=(M * K, nb1 * M * K), sB=(N * K, 0),
              sC=(M * ldc, nb1 * M * ldc), bias=_bf(N, seed=12), alpha=0.5)
    R.gemm(A, Bm, C, M, N, K, lda, ldb, ldc, **kw)
    res = G.gemm(A, Bm, C, M, N, K, lda, ldb, ldc, **kw)
    _check(res, C[..., :N], "batched")
    exact = 0.5 * (torch.einsum("xymk,ynk->xymn", a.double(), b.double()) + kw["bias"].double())
    assert torch.allclose(res.c, exact, rtol=1e-14, atol=0)


def test_gemm64_skew():
    T, H, Bz, hd = 13, 2, 3, 16
    d = H * hd
    q, k = _bf(Bz, T, d, seed=13), _bf(Bz, T, d, seed=14)
    ldp, ldt = 32, 16
    bd = _bf(H, Bz, T, ldp, seed=15)
    kw = dict(nb1=H, nb2=Bz, sA=(hd, T * d), sB=(hd, T * d), sC=(Bz * T * ldt, T * ldt), R=bd, ldr=ldp,
              sR=(Bz * T * ldp, T * ldp), skew_r=T, alpha=0.125, beta=1.0)
    sc = torch.zeros(H, Bz, T, ldt)
    R.gemm(q, k, sc, T, T, hd, d, d, ldt, **kw)
    res = G.gemm(q, k, sc, T, T, hd, d, d, ldt, **kw)
    _check(res, sc[..., :T].permute(1, 0, 2, 3), "skew")
    # element by element: BD row i, column (T - 1) - i + j
    i, j = 4, 9
    ac = (q[1, i].double().view(H, hd) * k[1, j].double().view(H, hd)).sum(-1)
    assert torch.allclose(res.c[1, :, i, j], 0.125 * ac + bd[:, 1, i, T - 1 - i + j].double(), rtol=1e-14)


def test_gemm64_accumulate_and_rowsum():
    M, N, K = 40, 24, 300
    A = _bf(K, 48, seed=16)[:, :M]  # MN-major A = dy^T with a padded row stride
    B = _bf(K, N, seed=17)
    C = torch.randn(M, N, generator=torch.Generator().manual_seed(18))
    rs = torch.full((M + 3,), -1.0)
    res = G.gemm(A, B, C, M, N, K, 48, N, N, a_kmajor=False, b_kmajor=False, accumulate=True, alpha=-1.0,
                 rowsum_a=rs, rowsum_scale=0.5)
    R.gemm(A, B, C, M, N, K, 48, N, N, a_kmajor=False, b_kmajor=False, accumulate=True, alpha=-1.0, rowsum_a=rs,
           rowsum_scale=0.5)
    _check(res, C, "accumulate")
    assert ((rs[:M].double() - res.rowsum).abs() <= 2e-6 * res.rowsum_mag).all()
    assert torch.equal(res.rowsum, -1.0 + 0.5 * A.double().sum(0))


CONV = [(2, 7, 9, 8, 5, (1, 1)), (2, 7, 9, 8, 5, (2, 2)), (1, 6, 11, 4, 6, (2, 1)), (1, 5, 4, 3, 4, (1, 2)),
        (1, 1, 1, 4, 4, (2, 2)), (1, 2, 3, 4, 4, (2, 2)), (2, 3, 2, 4, 4, (1, 1))]


@pytest.mark.parametrize("case", CONV)
def test_conv64_matches_torch_float64(case):
    B, T, Fq, Cin, Cout, stride = case
    x, w = _bf(B, T, Fq, Cin, seed=19), _bf(Cout, 3, 3, Cin, seed=20)
    xn = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    wn = w.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    yn = F.conv2d(xn, wn, None, stride, 1)
    y, ymag = G.conv3x3_fwd(x, w, stride)
    assert y.shape == (B, -(-T // stride[0]), -(-Fq // stride[1]), Cout)
    assert torch.allclose(y, yn.detach().permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    assert torch.allclose(ymag, F.conv2d(xn.detach().abs(), wn.detach().abs(), None, stride, 1).permute(0, 2, 3, 1))
    dy = _bf(*y.shape, seed=21)
    dyn = dy.double().permute(0, 3, 1, 2)
    yn.backward(dyn)
    dx, dxmag = G.conv3x3_dgrad(dy, w, x.shape, stride)
    To, Fo = y.shape[1], y.shape[2]
    opad = (T - (To - 1) * stride[0] - 1, Fq - (Fo - 1) * stride[1] - 1)
    dxt = F.conv_transpose2d(dyn, wn.detach(), None, stride, 1, opad)
    assert torch.allclose(dx, dxt.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    assert torch.allclose(dx, xn.grad.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    assert (dx.abs() <= dxmag * (1 + 1e-12)).all()
    dw0 = torch.randn(Cout, 3, 3, Cin, generator=torch.Generator().manual_seed(22))
    dw, dwmag = G.conv3x3_wgrad(dy, x, stride, dw0)
    assert torch.allclose(dw, dw0.double() + wn.grad.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    assert (dw.abs() <= dwmag * (1 + 1e-12)).all()
