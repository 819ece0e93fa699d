"""The GEMM's two epilogue warpgroups (csrc/gemm_tcgen05.cu) each serve one 64-row half of a tile, behind their own
acc_full / acc_empty handoff with the MMA warpgroup that stages those rows.  These cases put the last M tile at
M mod 128 = 1 (one valid row in half 0, none in half 1), 64 (half 1 empty) and 65 (one valid row in half 1), with K = 64
(one k-block of MMA per tile) and at least 8 tiles per CTA, so that a half whose rows are all out of range still has to
hand its staging buffer back in step with the other half.  They run on each instance the tile chooser picks (BN 64;
BN 128 single CTA; BN 128 on 2-CTA clusters whose last pair misses its odd tile), through every epilogue branch, the
fused skew residual and split-K accumulation with the bias-gradient row sums.

Each case is checked against float64 with the bounds of test_gpu_gemm_reference.py, and every non-accumulating case runs
twice: the two outputs must agree bit for bit."""
import pytest
import torch
from test_gpu_gemm_reference import (BF, BRANCHES, F32, TAU, TAU_ACC, EPS_SIG, _achieved, _achieved_c2,  # noqa: F401
                                     _assert_untouched, _epilogue_kw, _instance, _logical, _ops, _pair, _rand,
                                     _sentinel, _sig_achieved, _sms, _store)

pytestmark = pytest.mark.gpu

INSTANCES = [(64, 1), (128, 1), (128, 2)]
# (M mod 128, output dtype)
RESIDUES = [(1, BF), (64, F32), (65, BF), (65, F32)]


def _shape(bn, mc, r):
    """(M, N, tile_n): M = r mod 128, N ragged, at least 8 tiles (MC 2: tile pairs) per persistent CTA (cluster)."""
    if mc == 1:
        M, tm = 14 * 128 + r, 15         # 15 M tiles (odd, < 16: no pairing), the last one holding r rows
        slots = _sms()
    else:
        M, tm = 16 * 128 + r, 9          # 17 M tiles = 9 pairs: tile 16 holds r rows, tile 17 is missing
        slots = _sms() // 2
    tn = -(-8 * slots // tm)
    return M, tn * bn - 40, bn


@pytest.mark.parametrize("r,dt", RESIDUES, ids=["r%d_%s" % (r, "fp32" if dt == F32 else "bf16") for r, dt in RESIDUES])
@pytest.mark.parametrize("bn,mc", INSTANCES)
@pytest.mark.parametrize("branch", list(BRANCHES))
def test_ragged_half_every_branch(branch, bn, mc, r, dt, parity):
    spec = BRANCHES[branch]
    M, N, tile_n = _shape(bn, mc, r)
    assert _instance(M, N, tile_n) == (bn, mc)
    K = 64
    seed = 3 * r + bn + mc + len(branch)
    a, b = _rand((M, K), "randn", seed), _rand((N, K), "randn", seed + 7, 0.1)
    A, lda = _store(a, True)
    Bm, ldb = _store(b, dt == BF)
    kw = dict(_epilogue_kw(spec, M, N, seed), tile_n=tile_n, b_kmajor=dt == BF)
    ldc = N + 8
    outs = []
    for run in range(2):
        c = _sentinel((M + 1, ldc), dt)
        c2 = _sentinel((M + 1, ldc), BF) if spec.get("C2") else None
        if run == 0:
            out, ref = _pair(A, Bm, c, M, N, K, lda, ldb, ldc, C2=c2, **kw)
        else:
            _ops().gemm(A, Bm, c, M, N, K, lda, ldb, ldc, C2=c2, **kw)
            out = _logical(c, M, N, ldc)
        torch.cuda.synchronize()
        _assert_untouched(c, out, "C")
        o2 = None
        if c2 is not None:
            o2 = _logical(c2, M, N, ldc)
            _assert_untouched(c2, o2, "C2")
        outs.append((out, o2))
    assert torch.equal(outs[0][0], outs[1][0]), "two runs of the same call differ"
    worst = _achieved(outs[0][0], ref, bf16=dt == BF)
    if outs[0][1] is not None:
        assert torch.equal(outs[0][1], outs[1][1]), "two runs of the same call differ in C2"
        worst = max(worst, _achieved_c2(outs[0][1], ref))
    name = "ragged half %-10s BN%d MC%d M%%128=%d %s out" % (branch, bn, mc, r, "fp32" if dt == F32 else "bf16")
    parity(name + " (err / mag)", worst, TAU)
    if spec.get("act") in (2, 4):
        parity(name + " (sigmoid approximation error)", _sig_achieved(outs[0][0], ref, TAU, dt == BF), EPS_SIG)


@pytest.mark.parametrize("T", [64, 65])
def test_ragged_half_skew_batched(T, parity):
    """Batched scores with the fused skew residual, one 128 x 128 tile per (head, utterance), 8 per CTA: T = 64 leaves
    half 1 of every tile empty, T = 65 gives it one row."""
    H, K = 8, 64
    Bz = _sms()
    d = H * K
    q, k = _rand((Bz * T, d), "randn", T), _rand((Bz * T, d), "randn", T + 1)
    ldp, ldt = (2 * T - 1 + 7) // 8 * 8, (T + 7) // 8 * 8
    bd = _rand((H, Bz, T, ldp), "randn", T + 2)
    kw = dict(nb1=H, nb2=Bz, sA=(K, T * d), sB=(K, T * d), sC=(Bz * T * ldt, T * ldt), R=bd, ldr=ldp,
              sR=(Bz * T * ldp, T * ldp), skew_r=T, alpha=0.125, tile_n=128)
    S = _sentinel((H, Bz, T, ldt), BF)
    out, ref = _pair(q, k, S, T, T, K, d, d, ldt, **kw)
    S2 = _sentinel((H, Bz, T, ldt), BF)
    _ops().gemm(q, k, S2, T, T, K, d, d, ldt, **kw)
    torch.cuda.synchronize()
    _assert_untouched(S, out, "scores")
    assert torch.equal(S[..., :T], S2[..., :T]), "two runs of the same call differ"
    parity("ragged half skew H=%d B=%d T'=%d hd=%d (err / mag)" % (H, Bz, T, K), _achieved(out, ref, bf16=True), TAU)


@pytest.mark.parametrize("r", [1, 64, 65])
@pytest.mark.parametrize("bn,mc", INSTANCES)
def test_ragged_half_accumulate_rowsum(bn, mc, r, parity):
    """fp32 accumulate (one K split at K = 64) with the bias-gradient row sums of the MN-major A operand."""
    M, N, tile_n = _shape(bn, mc, r)
    assert _instance(M, N, tile_n, accumulate=True) == (bn, mc)
    K = 64
    dy, xx = _rand((K, M), "randn", M + r), _rand((K, N), "randn", M + r + 1)
    A, lda = _store(dy.t(), False)
    Bm, ldb = _store(xx.t(), False)
    C = torch.randn(M, N, device="cuda")
    gb = torch.randn(M + 5, device="cuda")
    tail = gb[M:].clone()
    out, ref = _pair(A, Bm, C, M, N, K, lda, ldb, N, a_kmajor=False, b_kmajor=False, accumulate=True, rowsum_a=gb,
                     tile_n=tile_n)
    torch.cuda.synchronize()
    assert torch.equal(gb[M:], tail), "row sums written past M"
    name = "ragged half accumulate BN%d MC%d M%%128=%d" % (bn, mc, r)
    parity(name + " C (err / mag)", _achieved(out, ref, bf16=False), TAU_ACC)
    parity(name + " row sums (err / mag)", float(((gb[:M].double() - ref.rowsum).abs() / ref.rowsum_mag).max()), TAU_ACC)
