"""GPU: every dropout path of the kernels against the host statement of the counter RNG (oracle/dropout_rng.py) and
against the per-op oracle (oracle/ops_ref.py) with the same mask.

Each case asserts (a) the mask read back from the kernel equals keep(seed + device seed, logical index, p) exactly,
wherever the value before dropout is non-zero, and (b) the outputs match ops_ref at the tolerance of the kernel's
dropout-0 test.  Every case runs without a device seed and with ops.set_seed_tensor holding 2^64 - 5, so the kernels'
seed + *seed_ptr wraps modulo 2^64."""
import numpy as np
import pytest
import torch

from oracle import dropout_rng as RNG
from oracle import ops_ref

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


@pytest.fixture(params=[0, 2 ** 64 - 5], ids=["no_device_seed", "device_seed"])
def dseed(request, dev):
    """The device seed of the case (0 = none installed); installed in both ops and ops_ref, removed afterwards."""
    from espresso_b200 import ops

    v = request.param
    t = torch.tensor([v - 2 ** 64 if v >= 2 ** 63 else v], dtype=torch.int64)
    ops.set_seed_tensor(t.to(dev) if v else None)
    ops_ref.set_seed_tensor(t if v else None)
    yield v
    ops.set_seed_tensor(None)
    ops_ref.set_seed_tensor(None)


def _keep(seed, dseed, shape, p, ld=None):
    """Expected keep mask of a row-major [..., cols] block with logical row stride ld (default: cols)."""
    cols = shape[-1]
    rows = int(np.prod(shape[:-1]))
    idx = RNG.row_major_index(rows, cols, ld)
    return RNG.keep_mask(RNG.combine_seed(seed, dseed), idx, p).view(*shape)


def _check_mask(out, before, keep, what):
    """(a): the kernel's output is zero exactly where the expected mask drops, wherever the value before dropout is not."""
    out, before = out.float().cpu(), before.float().cpu()
    nz = before != 0
    assert nz.float().mean() > 0.3, what            # enough observable elements
    got = out != 0
    bad = (got != keep) & nz
    assert not bad.any(), "%s: %d mask mismatches, first at %s" % (what, int(bad.sum()), bad.nonzero()[0].tolist())


def _err(a, b):
    return (a.float().cpu() - b.float().cpu()).abs().max().item()


# ------------------------------------------------------------------------------------------ GEMM epilogue
@pytest.mark.parametrize("N", [264, 1001, 30, 19, 7, 522])   # N mod 4 = 0, 1, 2, 3, 3, 2: the scalar branch runs for N % 4 != 0
@pytest.mark.parametrize("tile_n", [0, 64, 128, 256, 512])    # 512: 2-CTA clusters with B-tile multicast
def test_gemm_dropout(dev, dseed, tile_n, N):
    from espresso_b200 import ops

    M, K, p, seed = 333, 136, 0.25, 0x5EED0000 + N       # ragged M (not a multiple of the 128-row tile)
    g = torch.Generator().manual_seed(N + tile_n)
    a = torch.randn(M, K, generator=g).bfloat16()
    w = (torch.randn(N, K, generator=g) * 0.2).bfloat16()
    bias = torch.randn(N, generator=g).bfloat16()
    res = torch.randn(M, N, generator=g).bfloat16()
    ldc = (N + 7) // 8 * 8                                # padded output rows: the index uses N, not ldc
    ad, wd, bd, rd = a.to(dev), w.to(dev), bias.to(dev), torch.zeros(M, ldc, dtype=BF, device=dev)
    rd[:, :N] = res.to(dev)
    keep = _keep(seed, dseed, (M, N), p)
    for mode, act in ((1, ops.ACT_SILU), (1, ops.ACT_RELU), (2, ops.ACT_SILU), (2, ops.ACT_RELU)):
        kw = dict(bias=bd, act=act, drop_p=p, drop_mode=mode, seed=seed, tile_n=tile_n)
        # (a) mask: fp32 output without residual, against the same epilogue at p = 0.  Mode 2 drops before the
        # activation: only positive pre-activations are observable (SiLU of a large negative x * scale is 0 in fp32)
        y = torch.empty(M, ldc, device=dev)
        y0 = torch.empty(M, ldc, device=dev)
        ops.gemm(ad, wd, y, M, N, K, K, K, ldc, **kw)
        ops.gemm(ad, wd, y0, M, N, K, K, K, ldc, **dict(kw, drop_p=0.0, drop_mode=0))
        before = y0[:, :N] if mode == 1 else y0[:, :N].clamp(min=0)
        _check_mask(y[:, :N], before, keep, "gemm tile_n=%d N=%d mode=%d act=%d" % (tile_n, N, mode, act))
        # (b) values: bias + activation + C2 side output + scaled residual, bf16 output
        c = torch.zeros(M, ldc, dtype=BF, device=dev)
        c2 = torch.zeros(M, ldc, dtype=BF, device=dev)
        ops.gemm(ad, wd, c, M, N, K, K, K, ldc, C2=c2, R=rd, ldr=ldc, alpha=0.5, beta=1.0, **kw)
        cr = torch.zeros(M, ldc, dtype=BF)
        c2r = torch.zeros(M, ldc, dtype=BF)
        ops_ref.gemm(a, w, cr, M, N, K, K, K, ldc, C2=c2r, R=rd.cpu(), ldr=ldc, alpha=0.5, beta=1.0, **dict(kw, bias=bias))
        sc = max(1.0, cr.float().abs().max().item())
        assert _err(c[:, :N], cr[:, :N]) <= 0.02 * sc + 1e-2, (mode, act, _err(c, cr))
        assert _err(c2[:, :N], c2r[:, :N]) < 0.06


def test_gemm_dropout_batched(dev, dseed):
    """Batch dims (nb1, nb2): the index is (bt * M + m) * N + n with bt = b2 * nb1 + b1."""
    from espresso_b200 import ops

    nb1, nb2, M, N, K, p, seed = 3, 2, 77, 45, 64, 0.3, 4321
    ldc = 48
    g = torch.Generator().manual_seed(11)
    a = torch.randn(nb2, nb1, M, K, generator=g).bfloat16()
    b = (torch.randn(nb2, nb1, N, K, generator=g) * 0.3).bfloat16()
    kw = dict(nb1=nb1, nb2=nb2, sA=(M * K, nb1 * M * K), sB=(N * K, nb1 * N * K), sC=(M * ldc, nb1 * M * ldc),
              drop_p=p, drop_mode=1, seed=seed)
    y = torch.zeros(nb2, nb1, M, ldc, device=dev)
    y0 = torch.zeros(nb2, nb1, M, ldc, device=dev)
    ops.gemm(a.to(dev), b.to(dev), y, M, N, K, K, K, ldc, **kw)
    ops.gemm(a.to(dev), b.to(dev), y0, M, N, K, K, K, ldc, **dict(kw, drop_p=0.0, drop_mode=0))
    _check_mask(y[..., :N], y0[..., :N], _keep(seed, dseed, (nb2, nb1, M, N), p), "batched gemm")
    yr = torch.zeros(nb2, nb1, M, ldc)
    ops_ref.gemm(a, b, yr, M, N, K, K, K, ldc, **kw)
    assert _err(y, yr) <= 2e-3 * K ** 0.5 * RNG.scale(p) + 1e-3


@pytest.mark.parametrize("p", [1e-6, 0.9999])
def test_gemm_dropout_p_edges(dev, dseed, p):
    """p = 1e-6 quantises to thresh 0 (identity, scale exactly 1); p = 0.9999 keeps a few elements at scale 65536/7."""
    from espresso_b200 import ops

    M, N, K, seed = 600, 1000, 64, 77
    g = torch.Generator().manual_seed(5)
    a, w = torch.randn(M, K, generator=g).bfloat16(), torch.randn(N, K, generator=g).bfloat16()
    y = ops.linear(a.to(dev), w.to(dev), out_dtype=torch.float32, drop_p=p, drop_mode=1, seed=seed)
    y0 = ops.linear(a.to(dev), w.to(dev), out_dtype=torch.float32)
    keep = _keep(seed, dseed, (M, N), p)
    _check_mask(y, y0, keep, "gemm p=%g" % p)
    k = keep.to(dev)
    sc = RNG.scale(p)
    assert sc == float(np.float32(65536.0 / (65536 - RNG.thresh(p))))
    assert torch.equal(y[k], y0[k] * sc)   # fp32 epilogue: the kept values are exactly acc * scale
    if p < 1e-3:
        assert keep.all() and sc == 1.0 and torch.equal(y, y0)


# ------------------------------------------------------------------------------------------ esp_dropout
@pytest.mark.parametrize("N", [256, 264])      # 264: 33 vectors of 8 per row, not a power of two (the row / column split)
@pytest.mark.parametrize("p", [0.1, 1e-6, 0.9999])
def test_dropout_kernel_mask_and_values(dev, dseed, N, p):
    from espresso_b200 import ops

    R, ld, seed, scale = 1000, N + 16, 31337, 0.5
    g = torch.Generator().manual_seed(N)
    xs = torch.randn(R, ld, generator=g).bfloat16()
    x = xs[:, :N]                               # row stride ld > N: the index uses N
    y = ops.dropout(xs.to(dev)[:, :N], p, seed, scale=scale)
    _check_mask(y, x, _keep(seed, dseed, (R, N), p), "dropout N=%d p=%g" % (N, p))
    yr = ops_ref.dropout(x, p, seed, scale=scale)
    assert torch.equal(y.cpu(), yr)              # same fp32 products, same bf16 rounding


# ------------------------------------------------------------------------------------------ LayerNorm
def test_layer_norm_dropout(dev, dseed):
    from espresso_b200 import ops

    B, T, d, p = 3, 70, 256, 0.2
    R = B * T
    lens = torch.tensor([70, 41, 1], dtype=torch.int32)
    g = torch.Generator().manual_seed(3)
    x = torch.randn(R, d, generator=g).bfloat16()
    gam = (1 + 0.1 * torch.randn(d, generator=g)).bfloat16()
    bet = (3 + 0.1 * torch.randn(d, generator=g)).bfloat16()     # y away from 0: zeros mark dropped elements
    dy = torch.randn(R, d, generator=g).bfloat16()
    dres = torch.randn(R, d, generator=g).bfloat16()
    xd, gd, bd, ld_ = x.to(dev), gam.to(dev), bet.to(dev), lens.to(dev)
    y, mean, rstd = ops.layer_norm_fwd(xd, gd, bd, 1e-5, lens=ld_, T=T, drop_p=p, seed=901)
    y0, _, _ = ops.layer_norm_fwd(xd, gd, bd, 1e-5, lens=ld_, T=T)
    _check_mask(y.view(B, T, d)[0], y0.view(B, T, d)[0], _keep(901, dseed, (R, d), p)[:T], "layer_norm_fwd")
    yr, mr, rr = ops_ref.layer_norm_fwd(x, gam, bet, 1e-5, lens=lens, T=T, drop_p=p, seed=901)
    assert _err(y, yr) < 0.05 * RNG.scale(p)
    assert not y.view(B, T, d)[1, 41:].any() and not y.view(B, T, d)[2, 1:].any()
    # backward with the forward's mask (drop_p, seed) and the next module's masked copy (next_drop)
    for nd in (None, (0.1, 555, 0.5), (0.3, 556, 1.0)):
        ga, gb = torch.zeros(d, device=dev), torch.zeros(d, device=dev)
        gar, gbr = torch.zeros(d), torch.zeros(d)
        out = ops.layer_norm_bwd(dy.to(dev), xd, mean, rstd, gd, ga, gb, dres=dres.to(dev), lens=ld_, T=T, drop_p=p, seed=901,
                                 next_drop=nd)
        ref = ops_ref.layer_norm_bwd(dy, x, mean.cpu(), rstd.cpu(), gam, gar, gbr, dres=dres, lens=lens, T=T, drop_p=p, seed=901,
                                     next_drop=nd)
        dx, dxr = (out[0], ref[0]) if nd else (out, ref)
        sc = max(1.0, dxr.float().abs().max().item())
        assert _err(dx, dxr) < 2e-2 * sc, _err(dx, dxr)
        assert _err(ga, gar) < 2e-2 * max(1.0, gar.abs().max().item())
        assert _err(gb, gbr) < 2e-2 * max(1.0, gbr.abs().max().item())
        if nd:
            _check_mask(out[1], dx, _keep(nd[1], dseed, (R, d), nd[0]), "layer_norm_bwd2 next_drop")
            # the masked copy is dropout(bf16 dx) * scale on the GPU's own dx: exact
            assert torch.equal(out[1].cpu(), ops_ref.dropout(dx.cpu(), nd[0], nd[1], scale=nd[2]))


# ------------------------------------------------------------------------------------------ attention softmax
@pytest.mark.parametrize("causal", [False, True])
def test_attn_softmax_dropout(dev, dseed, causal):
    from espresso_b200 import ops

    H, B, T, p, seed = 3, 2, 203, 0.2, 77
    ld = (T + 7) // 8 * 8
    ldp = (2 * T - 1 + 7) // 8 * 8
    g = torch.Generator().manual_seed(9)
    s = (torch.randn(H, B, T, ld, generator=g) * 2).bfloat16()
    lens = None if causal else torch.tensor([T, 150], dtype=torch.int32)
    pr, pd = ops.attn_softmax_fwd(s.to(dev), T, None if lens is None else lens.to(dev), drop_p=p, seed=seed, causal=causal)
    prr, pdr = ops_ref.attn_softmax_fwd(s, T, lens, drop_p=p, seed=seed, causal=causal)
    keep = _keep(seed, dseed, (H, B, T, ld), p)
    nz = pr.cpu() != 0
    assert not ((pd.cpu() != 0) != keep)[nz].any()
    assert _err(pr, prr) < 1.5e-2 and _err(pd, pdr) < 1.5e-2 * RNG.scale(p)
    dpd = torch.randn(H, B, T, ld, generator=g).bfloat16()
    ds, dbd = ops.attn_softmax_bwd(pr, dpd.to(dev), T, ldp, drop_p=p, seed=seed)
    dsr, dbdr = ops_ref.attn_softmax_bwd(pr.cpu(), dpd, T, ldp, drop_p=p, seed=seed)
    sc = max(dsr.float().abs().max().item(), 1e-3)
    assert _err(ds, dsr) / sc < 2e-2 and _err(dbd, dbdr) / sc < 2e-2


# ------------------------------------------------------------------------------------------ fused attention
def _attn_inputs(B, T, H, seed):
    g = torch.Generator().manual_seed(seed)
    d = H * 64
    qkv = (torch.randn(B * T, 3 * d, generator=g) * 0.7).bfloat16()
    qu = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16()
    qv = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16()
    pos = (torch.randn(2 * T - 1, d, generator=g) * 0.7).bfloat16()
    return qu, qv, qkv, pos


ATTN_SHAPES = [(2, 25, 2, [25, 1]), (3, 129, 2, [129, 128, 1]), (3, 250, 4, [250, 160, 1]), (2, 407, 2, [407, 1])]


@pytest.mark.parametrize("B,T,H,lens", ATTN_SHAPES)
def test_attn_fused_dropout(dev, dseed, B, T, H, lens):
    """Forward: the mask of pd and pd / ctx against the fp32 statement with that mask.  Backward: dS, dBD, dK, dV against
    ops_ref.attn_fused_bwd (the mask regenerated from the same seed)."""
    from espresso_b200 import ops

    p, seed = 0.1, 0xABCDEF + T
    d = H * 64
    qu, qv, qkv, pos = _attn_inputs(B, T, H, T)
    k, v = qkv[:, d:2 * d], qkv[:, 2 * d:]
    lens_t = torch.tensor(lens, dtype=torch.int32)
    qkvd = qkv.to(dev)
    ctx, pr, pd = ops.attn_fused_fwd(qu.to(dev), qv.to(dev), qkvd[:, d:2 * d], qkvd[:, 2 * d:], pos.to(dev), B, T, H, lens_t.to(dev),
                                     drop_p=p, seed=seed)
    torch.cuda.synchronize()
    rc, rp, rpd = ops_ref.attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens_t, drop_p=p, seed=seed)
    ld = pr.shape[-1]
    keep = _keep(seed, dseed, (H, B, T, ld), p)[..., :T]
    nz = pr.cpu()[..., :T] != 0
    bad = ((pd.cpu()[..., :T] != 0) != keep) & nz
    assert not bad.any(), int(bad.sum())
    perr, pderr, cerr = _err(pr[..., :T], rp[..., :T]), _err(pd[..., :T], rpd[..., :T]), _err(ctx, rc)
    print("attn fused dropout B=%d T=%d H=%d: |dP| %.2e |dPd| %.2e |dctx| %.2e" % (B, T, H, perr, pderr, cerr))
    assert perr < 1.5e-2 and pderr < 1.5e-2 * RNG.scale(p)
    assert cerr < 2e-2 * max(1.0, rc.float().abs().max().item())
    # backward
    g = torch.Generator().manual_seed(T + 1)
    dctx = (torch.randn(B * T, d, generator=g) * 0.5).bfloat16()
    ldp = (2 * T - 1 + 7) // 8 * 8
    dqkv = torch.zeros(B * T, 3 * d, device=dev, dtype=BF)
    dS, dBD = ops.attn_fused_bwd(dctx.to(dev), ctx, qu.to(dev), qkvd[:, 2 * d:], pr, pd, B, T, H, ldp, dqkv[:, d:2 * d],
                                 dqkv[:, 2 * d:], p, seed)
    torch.cuda.synchronize()
    dk_r, dv_r = torch.empty(B * T, d, dtype=BF), torch.empty(B * T, d, dtype=BF)
    dS_r, dBD_r = ops_ref.attn_fused_bwd(dctx, ctx.cpu(), qu, v, pr.cpu(), pd.cpu(), B, T, H, ldp, dk_r, dv_r, p, seed)
    sc = max(dS_r.float().abs().max().item(), 1e-3)
    dk, dks = dqkv[:, d:2 * d].float().cpu(), max(dk_r.float().abs().max().item(), 1e-3)
    # The kernel's softmax row term is D = dctx . ctx with ctx the dropped, rescaled context rounded to bf16.  The single
    # key of a one-frame utterance is attended with probability 1 by all T query rows, so its exact dS (and dK) is 0 and
    # the kernel returns the bf16 rounding residue of D summed over T rows (a few % of max |dK| at T ~ 400): bounded
    # separately, every other key tightly.
    solo = torch.zeros(B, T, dtype=torch.bool)
    for b, n in enumerate(lens):
        solo[b, 0] = n == 1
    solo = solo.reshape(-1)
    e = (_err(dS, dS_r) / sc, _err(dBD, dBD_r) / sc, _err(dk[~solo], dk_r[~solo]) / dks,
         _err(dqkv[:, 2 * d:], dv_r) / max(dv_r.float().abs().max().item(), 1e-3))
    e_solo = _err(dk[solo], dk_r[solo]) / dks
    print("attn fused bwd dropout: dS %.2e dBD %.2e dK %.2e dV %.2e; dK of one-frame utterances %.2e" % (e + (e_solo,)))
    assert max(e) < 2e-2, e
    assert e_solo < 0.1, e_solo


# ------------------------------------------------------------------------------------------ embedding
def test_embed_dropout(dev, dseed):
    from espresso_b200 import ops

    V, d, B, U, p, seed, pad = 300, 256, 4, 37, 0.1, 2024, 1
    g = torch.Generator().manual_seed(4)
    E = (torch.randn(V, d, generator=g) * 0.5).bfloat16()
    E[pad] = 0
    pos = torch.randn(U, d, generator=g).bfloat16()
    tok = torch.randint(4, V, (B * U,), generator=g, dtype=torch.int32)
    tok[U - 5:U] = pad
    x = ops.embed_fwd(tok.to(dev), E.to(dev), pos.to(dev), U, 8.0, pad, drop_p=p, seed=seed)
    x0 = ops.embed_fwd(tok.to(dev), E.to(dev), pos.to(dev), U, 8.0, pad)
    _check_mask(x, x0, _keep(seed, dseed, (B * U, d), p), "embed_fwd")
    assert torch.equal(x.cpu(), ops_ref.embed_fwd(tok, E, pos, U, 8.0, pad, drop_p=p, seed=seed))
    dx = torch.randn(B * U, d, generator=g).bfloat16()
    dE = torch.zeros(V, d, device=dev)
    dEr = torch.zeros(V, d)
    ops.embed_bwd(tok.to(dev), dx.to(dev), dE, 8.0, pad, drop_p=p, seed=seed)
    ops_ref.embed_bwd(tok, dx, dEr, 8.0, pad, drop_p=p, seed=seed)
    assert _err(dE, dEr) < 1e-4 * max(1.0, dEr.abs().max().item())
    assert not dE[pad].any()
