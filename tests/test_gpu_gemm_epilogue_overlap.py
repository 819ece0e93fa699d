"""The GEMM's epilogue warpgroup (64- and 128-wide tiles of csrc/gemm_tcgen05.cu) hands every tile through one staging
buffer while the MMA warpgroups already run the next tile.  These shapes make that handoff as tight as it gets: K = 64 or
128 (one or two k-blocks of MMA per tile) and at least 8 tiles per CTA, with ragged M and N, on each instance the tile
chooser picks (BN 64; BN 128 single CTA; BN 128 on 2-CTA clusters whose last pair misses its odd tile), through every
epilogue branch, the implicit-GEMM convolutions (modes 1 and 2) and split-K with the fused bias-gradient row sums.

Each case is checked against float64 with the bounds of test_gpu_gemm_reference.py.  Each non-accumulating case runs
twice, and the two outputs must agree bit for bit: a tile staged over one the epilogue has not finished reading would
show up as a difference."""
import pytest
import torch
from test_gpu_gemm_reference import (BF, BRANCHES, F32, TAU, TAU_ACC, EPS_SIG, _achieved, _achieved_c2,  # noqa: F401
                                     _assert_untouched, _env, _epilogue_kw, _g64, _instance, _ksplit, _logical, _ops,
                                     _pair, _rand, _sentinel, _sig_achieved, _sms, _store, _tau_reached)

pytestmark = pytest.mark.gpu

INSTANCES = [(64, 1), (128, 1), (128, 2)]


def _shape(bn, mc):
    """(M, N, tile_n): ragged M and N with at least 8 tiles (MC 2: tile pairs) per persistent CTA (cluster)."""
    if mc == 1:
        M, tm = 1900, 15                 # 15 M tiles (odd, < 16: no pairing), the last one ragged
        slots = _sms()
    else:
        M, tm = 2126, 9                  # 17 M tiles = 9 pairs, the 9th without its odd tile
        slots = _sms() // 2
    tn = -(-8 * slots // tm)
    return M, tn * bn - 40, bn


def _run_twice(A, Bm, M, N, K, lda, ldb, ldc, dt, c2, kw):
    """The kernel once more into fresh sentinel buffers: (C, C2) logical views."""
    c = _sentinel((M + 1, ldc), dt)
    c2b = _sentinel((M + 1, ldc), BF) if c2 else None
    _ops().gemm(A, Bm, c, M, N, K, lda, ldb, ldc, C2=c2b, **kw)
    return _logical(c, M, N, ldc), (_logical(c2b, M, N, ldc) if c2 else None)


@pytest.mark.parametrize("K", [64, 128])
@pytest.mark.parametrize("bn,mc", INSTANCES)
@pytest.mark.parametrize("branch", list(BRANCHES))
def test_many_short_tiles_every_branch(branch, bn, mc, K, parity):
    spec = BRANCHES[branch]
    M, N, tile_n = _shape(bn, mc)
    assert _instance(M, N, tile_n) == (bn, mc)
    dt = F32 if K == 64 else BF
    seed = 7 * K + bn + mc + len(branch)
    a, b = _rand((M, K), "randn", seed), _rand((N, K), "randn", seed + 7, 0.1)
    A, lda = _store(a, True)
    Bm, ldb = _store(b, K == 128)
    kw = dict(_epilogue_kw(spec, M, N, seed), tile_n=tile_n, b_kmajor=K == 128)
    ldc = N + 8
    c = _sentinel((M + 1, ldc), dt)
    c2 = _sentinel((M + 1, ldc), BF) if spec.get("C2") else None
    out, ref = _pair(A, Bm, c, M, N, K, lda, ldb, ldc, C2=c2, **kw)
    again, again2 = _run_twice(A, Bm, M, N, K, lda, ldb, ldc, dt, c2 is not None, kw)
    torch.cuda.synchronize()
    _assert_untouched(c, out, "C")
    assert torch.equal(out, again), "two runs of the same call differ"
    worst = _achieved(out, ref, bf16=dt == BF)
    if c2 is not None:
        o2 = _logical(c2, M, N, ldc)
        _assert_untouched(c2, o2, "C2")
        assert torch.equal(o2, again2), "two runs of the same call differ in C2"
        worst = max(worst, _achieved_c2(o2, ref))
    name = "short tiles %-10s BN%d MC%d K=%d %s out" % (branch, bn, mc, K, "fp32" if dt == F32 else "bf16")
    parity(name + " (err / mag)", worst, TAU)
    if spec.get("act") in (2, 4):
        parity(name + " (sigmoid approximation error)", _sig_achieved(out, ref, TAU, dt == BF), EPS_SIG)


@pytest.mark.parametrize("K", [64, 128])
def test_many_short_tiles_skew_batched(K, parity):
    """Batched scores with the fused skew residual: 8 heads x (one per SM) utterances of 100 frames, hd = K."""
    H, T = 8, 100
    Bz = _sms()  # one 128 x 128 tile per (head, utterance): 8 per CTA
    d = H * K
    q, k = _rand((Bz * T, d), "randn", K), _rand((Bz * T, d), "randn", K + 1)
    ldp, ldt = (2 * T - 1 + 7) // 8 * 8, (T + 7) // 8 * 8
    bd = _rand((H, Bz, T, ldp), "randn", K + 2)
    kw = dict(nb1=H, nb2=Bz, sA=(K, T * d), sB=(K, T * d), sC=(Bz * T * ldt, T * ldt), R=bd, ldr=ldp,
              sR=(Bz * T * ldp, T * ldp), skew_r=T, alpha=0.125)
    S = _sentinel((H, Bz, T, ldt), BF)
    out, ref = _pair(q, k, S, T, T, K, d, d, ldt, **kw)
    S2 = _sentinel((H, Bz, T, ldt), BF)
    _ops().gemm(q, k, S2, T, T, K, d, d, ldt, **kw)
    torch.cuda.synchronize()
    _assert_untouched(S, out, "scores")
    assert torch.equal(S[..., :T], S2[..., :T]), "two runs of the same call differ"
    parity("short tiles skew H=%d B=%d T'=%d hd=%d (err / mag)" % (H, Bz, T, K), _achieved(out, ref, bf16=True), TAU)


# B, T, F, Cin, Cout, stride: about 9 (fwd) and more (dgrad parity classes) 128-row tiles per CTA at 576 / 1152 reduction
CONV = [(2, 1000, 80, 64, 64, (1, 1)), (1, 1800, 80, 64, 128, (2, 2))]


@pytest.mark.parametrize("case", CONV, ids=lambda c: "B%d_T%d_F%d_%dto%d_s%d%d" % (c[:5] + c[5]))
def test_conv3x3_many_tiles(case, parity):
    ops, g64 = _ops(), _g64()
    B, T, Fq, Cin, Cout, stride = case
    x = _rand((B, T, Fq, Cin), "randn", T)
    w = _rand((Cout, 3, 3, Cin), "randn", T + 1, (9 * Cin) ** -0.5)
    y = ops.conv3x3_fwd(x, w, stride)
    y_again = ops.conv3x3_fwd(x, w, stride)
    y64, ymag = g64.conv3x3_fwd(x, w, stride)
    dy = _rand(tuple(y.shape), "randn", T + 2)
    dx = ops.conv3x3_dgrad(dy, w, x.shape, stride)
    dx_again = ops.conv3x3_dgrad(dy, w, x.shape, stride)
    dx64, dxmag = g64.conv3x3_dgrad(dy, w, x.shape, stride)
    dw = torch.randn(Cout, 3, 3, Cin, device="cuda")
    dw64, dwmag = g64.conv3x3_wgrad(dy, x, stride, dw)
    ops.conv3x3_wgrad(dy, x, dw, stride)
    torch.cuda.synchronize()
    assert torch.equal(y, y_again) and torch.equal(dx, dx_again), "two runs of the same convolution differ"
    name = "short tiles conv3x3 B%d T%d F%d %d->%d stride %s" % (B, T, Fq, Cin, Cout, stride)
    parity(name + " fwd (err / mag)", _tau_reached(y, y64, ymag, None, bf16=True), TAU)
    parity(name + " dgrad (err / mag)", _tau_reached(dx, dx64, dxmag, None, bf16=True), TAU)
    parity(name + " wgrad (err / mag)", _tau_reached(dw, dw64, dwmag, None, bf16=False), TAU_ACC)


@pytest.mark.parametrize("M,N,K", [(1000, 600, 2048), (100, 64, 1024), (2000, 1000, 512)])
def test_splitk_rowsum_many_items(M, N, K, parity):
    """Split-K accumulate with the bias-gradient row sums, short K splits (4 k-blocks where the split allows it)."""
    ks = _ksplit(M, N, K)
    dy, xx = _rand((K, M), "randn", M + K), _rand((K, N), "randn", M + K + 1)
    A, lda = _store(dy.t(), False)
    Bm, ldb = _store(xx.t(), False)
    C = torch.randn(M, N, device="cuda")
    gb = torch.randn(M + 5, device="cuda")
    tail = gb[M:].clone()
    out, ref = _pair(A, Bm, C, M, N, K, lda, ldb, N, a_kmajor=False, b_kmajor=False, accumulate=True, rowsum_a=gb)
    torch.cuda.synchronize()
    assert torch.equal(gb[M:], tail), "row sums written past M"
    name = "short tiles wgrad M=%d N=%d K=%d ksplit %d" % (M, N, K, ks)
    parity(name + " C (err / mag)", _achieved(out, ref, bf16=False), TAU_ACC)
    parity(name + " row sums (err / mag)", float(((gb[:M].double() - ref.rowsum).abs() / ref.rowsum_mag).max()), TAU_ACC)
