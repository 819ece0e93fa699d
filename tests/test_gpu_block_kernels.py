"""GPU parity: every HBM-bound block kernel and the optimizer vs the oracle's per-op reference
(oracle/ops_ref.py, same signatures), through the C ABI."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _close(a, b, tol, what=""):
    a, b = a.float().cpu(), b.float().cpu()
    err = (a - b).abs().max().item()
    scale = max(b.abs().max().item(), 1e-3)
    assert err <= tol * scale, "%s: err %.4g vs scale %.4g" % (what, err, scale)


@pytest.mark.parametrize("R,d", [(37, 64), (1000, 512), (300, 256), (65, 1024)])
def test_layer_norm(dev, R, d):
    from espresso_b200 import ops
    from oracle import ops_ref as O

    torch.manual_seed(R)
    x = (torch.randn(R, d) * 2 + 0.5).to(BF)
    g = (1 + 0.2 * torch.randn(d)).to(BF)
    b = (0.2 * torch.randn(d)).to(BF)
    T = 25 if R % 25 == 0 else R
    lens = torch.tensor([T - 3] * (R // T), dtype=torch.int32) if R % 25 == 0 else None
    y, mean, rstd = ops.layer_norm_fwd(x.to(dev), g.to(dev), b.to(dev), lens=None if lens is None else lens.to(dev), T=T)
    yr, mr, rr = O.layer_norm_fwd(x, g, b, lens=lens, T=T)
    _close(y, yr, 0.01, "ln y")
    _close(mean, mr, 1e-4, "ln mean")
    _close(rstd, rr, 1e-4, "ln rstd")
    dy = torch.randn(R, d).to(BF)
    dres = torch.randn(R, d).to(BF)
    dg, db = torch.zeros(d, device=dev), torch.zeros(d, device=dev)
    dx = ops.layer_norm_bwd(dy.to(dev), x.to(dev), mean, rstd, g.to(dev), dg, db, dres=dres.to(dev),
                            lens=None if lens is None else lens.to(dev), T=T)
    dgr, dbr = torch.zeros(d), torch.zeros(d)
    dxr = O.layer_norm_bwd(dy, x, mr, rr, g, dgr, dbr, dres=dres, lens=lens, T=T)
    _close(dx, dxr, 0.02, "ln dx")
    _close(dg, dgr, 0.01, "ln dgamma")
    _close(db, dbr, 0.01, "ln dbeta")


def test_layer_norm_dropout_consistency(dev):
    """forward dropout mask == mask regenerated in backward (zeros line up), keep rate ~ 1-p."""
    from espresso_b200 import ops

    R, d, p = 400, 512, 0.1
    x = torch.randn(R, d, device=dev).to(BF)
    g = torch.ones(d, device=dev, dtype=BF)
    b = torch.full((d,), 3.0, device=dev, dtype=BF)  # keeps y away from 0 so zeros mark dropped elements
    y, mean, rstd = ops.layer_norm_fwd(x, g, b, drop_p=p, seed=77)
    dropped = (y == 0)
    assert abs(dropped.float().mean().item() - p) < 0.01
    dy = torch.ones(R, d, device=dev, dtype=BF)
    dg, db = torch.zeros(d, device=dev), torch.zeros(d, device=dev)
    ops.layer_norm_bwd(dy, x, mean, rstd, g, dg, db, drop_p=p, seed=77)
    # dbeta = sum_r mask/(1-p)  => counts of kept elements per column
    kept = (~dropped).float().sum(0) / (1 - p)
    assert (db - kept).abs().max().item() < 1e-2 * kept.max().item()


def test_colsum_dropout_mask_rows_qprep(dev):
    from espresso_b200 import ops
    from oracle import ops_ref as O

    torch.manual_seed(3)
    x = torch.randn(700, 1536).to(BF)
    acc = torch.ones(512, device=dev)
    ops.colsum(x.to(dev)[:, 512:1024], acc, scale=0.5)
    accr = torch.ones(512)
    O.colsum(x[:, 512:1024], accr, scale=0.5)
    _close(acc, accr, 2e-3, "colsum")
    y = ops.dropout(x.to(dev), 0.0, 1, scale=0.5)
    _close(y, O.dropout(x, 0.0, 1, scale=0.5), 1e-2, "scale")
    yd = ops.dropout(x.to(dev), 0.3, 5)
    keep = (yd != 0).float().mean().item()
    assert abs(keep - 0.7) < 0.01
    m = yd != 0
    _close(yd[m], (x.to(dev).float() / 0.7)[m], 1e-2, "dropout scale")
    # same (seed, index) stream as the GEMM epilogue: dropout(I @ x) masks must coincide
    eye = torch.eye(64, device=dev, dtype=BF)
    xs = torch.randn(64, 64, device=dev).to(BF) + 4
    via_gemm = ops.linear(eye, xs.t().contiguous(), drop_p=0.3, drop_mode=1, seed=5)
    via_kernel = ops.dropout(xs, 0.3, 5)
    assert torch.equal(via_gemm == 0, via_kernel == 0)
    # mask rows
    z = torch.randn(3, 20, 64).to(BF)
    lens = torch.tensor([20, 7, 1], dtype=torch.int32)
    zr = O.mask_rows_(z.clone(), lens)
    zg = ops.mask_rows_(z.to(dev).clone(), lens.to(dev))
    assert torch.equal(zg.cpu(), zr)
    # qprep
    q = x[:, :512]
    u, v = torch.randn(512).to(BF), torch.randn(512).to(BF)
    qu, qv = ops.qprep_fwd(x.to(dev)[:, :512], u.to(dev), v.to(dev), 0.125)
    qur, qvr = O.qprep_fwd(q, u, v, 0.125)
    _close(qu, qur, 1e-2, "qu")
    _close(qv, qvr, 1e-2, "qv")
    out = torch.zeros(700, 1536, device=dev, dtype=BF)
    ops.qprep_bwd(qu, qv, 0.125, out[:, :512])
    outr = torch.zeros(700, 1536, dtype=BF)
    O.qprep_bwd(qur, qvr, 0.125, outr[:, :512])
    _close(out, outr, 1e-2, "qprep bwd")


@pytest.mark.parametrize("T", [16, 61, 250, 305])
def test_attn_softmax(dev, T):
    from espresso_b200 import ops
    from oracle import ops_ref as O

    torch.manual_seed(T)
    H, B = 2, 3
    ld, ldp = (T + 7) // 8 * 8, (2 * T + 6) // 8 * 8
    s = (torch.randn(H, B, T, ld) * 3).to(BF)
    lens = torch.tensor([T, max(1, T - 5), max(1, T // 2)], dtype=torch.int32)
    p, pd = ops.attn_softmax_fwd(s.to(dev), T, lens.to(dev))
    pr, _ = O.attn_softmax_fwd(s, T, lens)
    _close(p[..., :T], pr[..., :T], 0.01, "softmax")
    assert not p[..., T:].any()
    p2, _ = ops.attn_softmax_fwd(s.to(dev), T, None)
    pr2, _ = O.attn_softmax_fwd(s, T, None)
    _close(p2[..., :T], pr2[..., :T], 0.01, "softmax nomask")
    dp = torch.randn(H, B, T, ld).to(BF)
    ds, dbd = ops.attn_softmax_bwd(p, dp.to(dev), T, ldp)
    dsr, dbdr = O.attn_softmax_bwd(p.cpu(), dp, T, ldp)
    _close(ds[..., :T], dsr[..., :T], 0.02, "softmax bwd")
    _close(dbd[..., : 2 * T - 1], dbdr[..., : 2 * T - 1], 0.02, "dBD scatter")
    # dropout variant: kept fraction, and backward uses the same mask
    p3, pd3 = ops.attn_softmax_fwd(s.to(dev), T, None, drop_p=0.2, seed=9)
    assert torch.equal(p3, p2)
    nz = p3[..., :T].float() > 1e-4
    keep = ((pd3[..., :T] != 0) & nz).float().sum().item() / nz.float().sum().item()
    assert abs(keep - 0.8) < 0.02
    ones = torch.ones(H, B, T, ld, device=dev, dtype=BF)
    ds3, _ = ops.attn_softmax_bwd(p3, ones, T, ldp, drop_p=0.2, seed=9)
    mask = (pd3[..., :T] != 0).float() / 0.8
    pf = p3[..., :T].float()
    expect = pf * (mask - (mask * pf).sum(-1, keepdim=True))
    sel = nz
    assert ((ds3[..., :T].float() - expect)[sel]).abs().max().item() < 0.02


@pytest.mark.parametrize("B,T,C,k", [(2, 50, 64, 31), (3, 200, 128, 31), (1, 7, 64, 3), (2, 65, 512, 31)])
def test_conv_module_kernels(dev, B, T, C, k):
    from espresso_b200 import ops
    from oracle import ops_ref as O

    torch.manual_seed(T + C)
    g = torch.randn(B, T, 2 * C).to(BF)
    w = (torch.randn(C, k) * 0.3).to(BF)
    y, stats = ops.glu_dwconv_fwd(g.to(dev), w.to(dev))
    yr, statsr = O.glu_dwconv_fwd(g, w)
    _close(y, yr, 0.02, "dwconv y")
    _close(stats, statsr, 0.02, "bn stats")
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    mr = ops.bn_finalize(stats, B * T, C, 1e-5, 0.1, rm, rv, True)
    rmr, rvr = torch.zeros(C), torch.ones(C)
    mrr = O.bn_finalize(statsr, B * T, C, 1e-5, 0.1, rmr, rvr, True)
    _close(mr, mrr, 0.02, "bn mean/rstd")
    _close(rm, rmr, 0.02, "running mean")
    _close(rv, rvr, 0.02, "running var")
    gm, bt = (1 + 0.2 * torch.randn(C)).to(BF), (0.2 * torch.randn(C)).to(BF)
    z = ops.bn_silu_fwd(y, mr, gm.to(dev), bt.to(dev))
    zr = O.bn_silu_fwd(y.cpu(), mr.cpu(), gm, bt)
    _close(z, zr, 0.02, "bn silu")
    mre = ops.bn_finalize(None, B * T, C, 1e-5, 0.1, rm, rv, False)  # eval: running stats
    _close(mre[0], rm, 1e-6, "eval mean")
    dz = torch.randn(B, T, C).to(BF)
    dgm, dbt = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    dy = ops.bn_silu_bwd(dz.to(dev), y, mr, gm.to(dev), bt.to(dev), dgm, dbt)
    dgmr, dbtr = torch.zeros(C), torch.zeros(C)
    dyr = O.bn_silu_bwd(dz, y.cpu(), mr.cpu(), gm, bt, dgmr, dbtr)
    _close(dy, dyr, 0.03, "bn bwd dy")
    _close(dgm, dgmr, 0.02, "bn dgamma")
    _close(dbt, dbtr, 0.02, "bn dbeta")
    dw = torch.zeros(C, k, device=dev)
    dg = ops.glu_dwconv_bwd(dy, g.to(dev), w.to(dev), dw)
    dwr = torch.zeros(C, k)
    dgr = O.glu_dwconv_bwd(dy.cpu(), g, w, dwr)
    _close(dg, dgr, 0.03, "dwconv dg")
    _close(dw, dwr, 0.03, "dwconv dw")


def test_optimizer_kernels(dev):
    from espresso_b200 import ops
    from oracle import ops_ref as O

    torch.manual_seed(0)
    n = 100003
    p32 = torch.randn(n)
    g = torch.randn(n + 8) * 3
    g[n] = 4.0  # tail: sample_size
    st = [dict(p32=p32.clone(), m=torch.zeros(n), v=torch.zeros(n), p16=torch.zeros(n, dtype=BF)) for _ in range(2)]
    gd = {k: v.to(dev) for k, v in st[0].items()}
    gg = g.to(dev)
    ss, ssr = torch.zeros(1, device=dev), torch.zeros(1)
    gn = torch.zeros(1, device=dev)
    for step in (1, 2, 3):
        ops.sumsq(gg[:n], ss)
        O.sumsq(g[:n], ssr)
        _close(ss, ssr, 1e-4, "sumsq")
        ops.adam_step(gd["p32"], gd["m"], gd["v"], gg, gd["p16"], 1e-2, 0.9, 0.98, 1e-8, 0.01, step, ss, denom_dev=gg[n:n + 1],
                      clip_norm=2.0, gnorm_out=gn)
        r = st[1]
        O.adam_step(r["p32"], r["m"], r["v"], g, r["p16"], 1e-2, 0.9, 0.98, 1e-8, 0.01, step, ssr, denom_dev=g[n:n + 1], clip_norm=2.0)
    _close(gd["p32"], st[1]["p32"], 1e-4, "adam p32")
    _close(gd["v"], st[1]["v"], 1e-3, "adam v")
    assert torch.equal(gd["p16"].cpu(), gd["p32"].cpu().to(BF))
    assert abs(gn.item() - ssr.item() ** 0.5 / 4.0) < 1e-3 * gn.item()
    x = torch.randn(1000, device=dev)
    y = torch.empty(1000, device=dev, dtype=BF)
    ops.cast_f32_bf16(x, y)
    assert torch.equal(y, x.to(BF))
    z = torch.empty(1000, device=dev)
    ops.cast_bf16_f32(y, z)
    assert torch.equal(z, y.float())


@pytest.mark.parametrize("R,C", [(5000, 64), (3333, 128), (777, 512)])
def test_bn_relu_channels_last(dev, R, C):
    """Conv-front BatchNorm2d + ReLU on NHWC activations (rows = B*T*F)."""
    from espresso_b200 import ops
    from oracle import ops_ref as O

    torch.manual_seed(R)
    x = (torch.randn(R, C) * 1.5 + 0.3).to(BF)
    st = ops.bn_stats(x.to(dev), C)
    _close(st, O.bn_stats(x, C), 1e-3, "bn_stats")
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    mr = ops.bn_finalize(st, R, C, 1e-5, 0.1, rm, rv, True)
    gm, bt = (1 + 0.2 * torch.randn(C)).to(BF), (0.2 * torch.randn(C)).to(BF)
    z = ops.bn_act_fwd(x.to(dev), mr, gm.to(dev), bt.to(dev), ops.BN_ACT_RELU)
    zr = O.bn_act_fwd(x, mr.cpu(), gm, bt, O.BN_ACT_RELU)
    _close(z, zr, 0.02, "bn relu")
    dz = torch.randn(R, C).to(BF)
    dg, db = torch.zeros(C, device=dev), torch.zeros(C, device=dev)
    dx = ops.bn_act_bwd(dz.to(dev), x.to(dev), mr, gm.to(dev), bt.to(dev), dg, db, ops.BN_ACT_RELU)
    dgr, dbr = torch.zeros(C), torch.zeros(C)
    dxr = O.bn_act_bwd(dz, x, mr.cpu(), gm, bt, dgr, dbr, O.BN_ACT_RELU)
    _close(dx, dxr, 0.03, "bn relu dx")
    _close(dg, dgr, 0.02, "bn relu dgamma")
    _close(db, dbr, 0.02, "bn relu dbeta")


@pytest.mark.parametrize("B,T,U,V", [(2, 5, 3, 8), (3, 40, 12, 50), (2, 30, 9, 5004), (2, 20, 0, 16)])
def test_rnnt_loss_vs_torchaudio(dev, B, T, U, V):
    """RNN-T loss + gradient vs the reference's own call (torchaudio.functional.rnnt_loss, fused log-softmax)."""
    from espresso_b200 import ops
    from oracle import ops_ref as O

    torch.manual_seed(T + V)
    U1 = U + 1
    ld = (V + 7) // 8 * 8
    x = torch.zeros(B, T, U1, ld)
    x[..., :V] = torch.randn(B, T, U1, V) * 1.5
    x = x.to(BF)
    t_lens = torch.tensor([T] + [max(1, T - 3 * i) for i in range(1, B)], dtype=torch.int32)
    u_lens = torch.tensor([U] + [max(0, U - 2 * i) for i in range(1, B)], dtype=torch.int32)
    tg = torch.randint(1, V, (B, max(U, 1)), dtype=torch.int32)
    loss, grad = ops.rnnt_loss(x.to(dev), V, t_lens.to(dev), u_lens.to(dev), tg.to(dev), 0, grad_scale=0.5)
    if U == 0:  # empty targets: the only path emits blank at every frame -> closed form
        lp = torch.log_softmax(x.float()[..., :V], -1)[:, :, 0, 0]
        ref = torch.stack([-lp[b, : t_lens[b]].sum() for b in range(B)])
        assert torch.allclose(loss.cpu(), ref, rtol=1e-5, atol=1e-3)
        return
    lr, gr = O.rnnt_loss(x, V, t_lens, u_lens, tg, 0, grad_scale=0.5)
    assert torch.allclose(loss.cpu(), lr, rtol=1e-5, atol=1e-3), (loss.cpu(), lr)
    g = grad.float().cpu()
    assert (g[..., :V] - gr.float()[..., :V]).abs().max().item() < 4e-3
    assert not g[..., V:].any()
    for b in range(B):  # cells outside the utterance's lattice get zero gradient
        assert not g[b, t_lens[b]:].any() and not g[b, :, u_lens[b] + 1:].any()


def test_joint_kernels(dev):
    from espresso_b200 import ops
    from oracle import ops_ref as O

    torch.manual_seed(2)
    B, T, U1, J = 3, 17, 6, 64
    e, d = torch.randn(B, T, J).to(BF), torch.randn(B, U1, J).to(BF)
    f = ops.joint_fwd(e.to(dev), d.to(dev))
    fr = O.joint_fwd(e, d)
    _close(f, fr, 0.01, "joint fwd")
    df = torch.randn(B, T, U1, J).to(BF)
    de, dd = ops.joint_bwd(df.to(dev), f)
    der, ddr = O.joint_bwd(df, fr)
    _close(de, der, 0.02, "joint denc")
    _close(dd, ddr, 0.01, "joint ddec")


# ---------------------------------------------------------------------------------------------------
# fused relative-position attention forward (csrc/attn_fused.cu) vs the fp32 statement of
# fairseq/modules/multihead_attention.py:788-897
# ---------------------------------------------------------------------------------------------------
def _attn_inputs(B, T, H, seed, dev, shared_pos=False):
    torch.manual_seed(seed)
    d = H * 64
    qkv = (torch.randn(B * T, 3 * d, device=dev) * 0.7).bfloat16()
    qu = (torch.randn(B * T, d, device=dev) * 0.3).bfloat16()
    qv = (torch.randn(B * T, d, device=dev) * 0.3).bfloat16()
    pos = (torch.randn(2 * T - 1, 64 if shared_pos else d, device=dev) * 0.7).bfloat16()
    return qu, qv, qkv[:, d:2 * d], qkv[:, 2 * d:], pos


@pytest.mark.parametrize("B,T,H,lens,shared", [
    (2, 25, 2, None, False),                 # one partial tile (1 s utterances)
    (3, 128, 2, [128, 77, 1], False),        # exactly one tile, padded keys, a single-key utterance
    (2, 129, 4, [129, 128], False),          # one row / key spills into a second tile
    (3, 407, 8, [407, 333, 150], False),     # the bench's typical T' (4 x 4 tiles)
    (1, 875, 2, None, False),                # 35 s utterance: 7 x 7 tiles
    (2, 200, 4, [200, 64], True),            # learned positions shared by all heads (head stride 0)
    (3, 250, 8, [250, 160, 77], False),      # the full-size parity fixture's shape (two tiles, second one ragged)
    (4, 64, 8, [64, 40, 33, 1], False),      # at most 64 keys: the second half-row warps see masked keys only
])
def test_attn_fused_fwd_vs_reference(dev, B, T, H, lens, shared):
    from espresso_b200 import ops
    from oracle import ops_ref

    qu, qv, k, v, pos = _attn_inputs(B, T, H, 100 + T, dev, shared)
    lens_t = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
    ctx, p, pd = ops.attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens_t)
    torch.cuda.synchronize()
    rc, rp, _ = ops_ref.attn_fused_fwd(qu.cpu(), qv.cpu(), k.cpu(), v.cpu(), pos.cpu(), B, T, H,
                                       None if lens is None else lens_t.cpu())
    assert pd is p
    perr = (p.float().cpu()[..., :T] - rp.float()[..., :T]).abs().max().item()
    cerr = (ctx.float().cpu() - rc.float()).abs().max().item()
    print("attn fused fwd B=%d T=%d H=%d: max |dP| %.2e, max |dctx| %.2e" % (B, T, H, perr, cerr))
    # probabilities are bf16 (<= 2^-9 relative on values <= 1); logits differ by the bf16 rounding of BD only
    assert perr < 1.5e-2, perr
    assert cerr < 2e-2 * max(1.0, rc.float().abs().max().item()), cerr
    ld = p.shape[-1]
    assert ld % 8 == 0 and (p[..., T:] == 0).all()
    assert torch.allclose(p.float()[..., :T].sum(-1), torch.ones(H, B, T, device=dev), atol=2e-2)
    if lens is not None:  # masked keys get exactly zero probability
        for b, l in enumerate(lens):
            assert (p[:, b, :, l:] == 0).all()
    # inference mode: same context, nothing else written
    ctx2, p2, _ = ops.attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens_t, save_probs=False)
    assert p2 is None and torch.equal(ctx2, ctx)


@pytest.mark.parametrize("B,T,lens,chunk,lw,rw,last,ctx", [
    (2, 203, [203, 150], 16, 1, 0, True, None),     # causal-ish chunks, one chunk of history
    (3, 407, [407, 333, 150], 40, 2, 1, False, None),  # training layout (coin decides which end is partial)
    (2, 130, None, 7, 0, 0, True, None),            # chunks smaller than a warp's column group, two key tiles
    (2, 64, [64, 20], 200, 0, 0, True, None),       # one chunk covers everything (mask is a no-op)
    (3, 250, [250, 160, 77], 0, 0, 0, True, (10, 3)),  # transformer_context band
    (2, 129, [129, 40], 0, 0, 0, True, (None, 0)),  # causal
    (2, 90, [90, 31], 30, 0, 0, True, None),        # rows of the short utterance whose visible chunk is all padding
])
def test_attn_fused_fwd_streaming_masks(dev, B, T, lens, chunk, lw, rw, last, ctx):
    """Per-row visible key ranges (chunk streaming, espresso/tools/utils.py:131-194; limited context,
    speech_transformer_encoder.py:250-263) inside the fused kernel vs the oracle's additive-mask statement."""
    from espresso_b200 import ops
    from espresso_b200.tools.utils import chunk_streaming_bounds, context_bounds
    from oracle import ops_ref

    H = 2
    qu, qv, k, v, pos = _attn_inputs(B, T, H, 300 + T, dev)
    np.random.seed(T)
    lo, hi = chunk_streaming_bounds(T, chunk, lw, rw, always_partial_in_last=last) if chunk else context_bounds(T, *ctx)
    lo_t, hi_t = torch.from_numpy(lo), torch.from_numpy(hi)
    lens_t = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
    out, p, _ = ops.attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens_t, key_bounds=(lo_t.to(dev), hi_t.to(dev)))
    torch.cuda.synchronize()
    rc, rp, _ = ops_ref.attn_fused_fwd(qu.cpu(), qv.cpu(), k.cpu(), v.cpu(), pos.cpu(), B, T, H,
                                       None if lens is None else lens_t.cpu(), key_bounds=(lo_t, hi_t))
    j = torch.arange(T)[None, :]
    hidden = (j < lo_t[:, None]) | (j >= hi_t[:, None])                       # [T, T]
    # rows whose visible keys are all padding normalise over the hidden keys (finite -1e4 mask): the reference's bf16
    # score arithmetic there is only reproduced approximately, compare everything else tightly
    L = torch.full((B,), T) if lens is None else torch.tensor(lens)
    vis = (~hidden)[None] & (j[None] < L[:, None, None])                      # [B, T, T]
    ok_rows = vis.any(-1)                                                      # [B, T]
    pg = p.float().cpu()[..., :T]
    perr = (pg - rp.float()[..., :T])[:, ok_rows].abs().max().item()
    cg, cr = out.float().cpu().view(B, T, -1), rc.float().view(B, T, -1)
    cerr = (cg - cr)[ok_rows].abs().max().item()
    assert perr < 1.5e-2 and cerr < 2e-2 * max(1.0, cr.abs().max().item()), (perr, cerr)
    # hidden keys carry exactly zero probability wherever a visible key exists
    assert (pg.permute(1, 2, 3, 0)[(ok_rows[:, :, None] & hidden[None])] == 0).all()
    assert torch.allclose(pg.sum(-1), torch.ones(H, B, T), atol=2e-2)
    if (~ok_rows).any():   # degenerate rows: still a proper distribution over the unpadded keys, never NaN
        assert torch.isfinite(cg).all()
        bad = (~ok_rows).nonzero()
        b0, i0 = bad[0].tolist()
        assert (pg[:, b0, i0, L[b0]:] == 0).all()


def test_attn_fused_fwd_dropout_stream_matches_softmax_kernels(dev):
    """The dropped probabilities use the same counter-RNG stream as esp_attn_softmax_fwd / _bwd (the backward pass
    regenerates the mask with esp_attn_softmax_bwd), and ctx == Pd v."""
    from espresso_b200 import ops

    B, T, H = 2, 203, 4
    qu, qv, k, v, pos = _attn_inputs(B, T, H, 7, dev)
    ctx, p, pd = ops.attn_fused_fwd(qu, qv, k, v, pos, B, T, H, None, drop_p=0.25, seed=4242)
    ld = p.shape[-1]
    # reference mask: the unfused kernel on arbitrary scores of the same shape with the same seed
    _, pd_ref = ops.attn_softmax_fwd(torch.zeros(H, B, T, ld, device=dev, dtype=torch.bfloat16), T, None, drop_p=0.25, seed=4242)
    keep_ref = pd_ref[..., :T] != 0
    keep = pd[..., :T] != 0
    nz = p[..., :T] != 0          # a probability that underflowed to 0 says nothing about its mask bit
    assert torch.equal(keep[nz], keep_ref[nz])
    kept = pd[..., :T][keep].float()
    assert torch.allclose(kept, (p[..., :T][keep].float() * (1 / 0.75)).bfloat16().float(), rtol=1e-2, atol=1e-6)
    assert abs(keep_ref.float().mean().item() - 0.75) < 0.01
    d = H * 64
    ref = torch.einsum("hbij,bjhe->bihe", pd[..., :T].float(), v.float().reshape(B, T, H, 64)).reshape(B * T, d)
    assert (ctx.float() - ref).abs().max().item() < 2e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("B,T,H,lens,drop", [(2, 250, 4, [250, 131], 0.0), (3, 64, 2, None, 0.0), (1, 407, 8, None, 0.0),
                                             (2, 129, 2, [129, 40], 0.0), (2, 203, 4, [203, 150], 0.25), (2, 300, 8, None, 0.1)])
def test_attn_fused_bwd(dev, B, T, H, lens, drop):
    """Score side of the attention backward in one kernel (csrc/attn_fused_bwd.cu) against the fp32 statement of the
    chain (oracle/ops_ref.py), which regenerates the dropout mask with the kernels' counter RNG (oracle/dropout_rng.py)."""
    from espresso_b200 import ops
    from oracle import ops_ref

    ops.set_seed_tensor(None)      # no device seed on either side (a trainer built by an earlier test installs one)
    ops_ref.set_seed_tensor(None)
    d = H * 64
    qu, qv, k, v, pos = _attn_inputs(B, T, H, 900 + T, dev)
    lens_t = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
    ctx, p, pd = ops.attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens_t, drop_p=drop, seed=99)
    g = torch.Generator(device="cpu").manual_seed(T)
    dctx = (torch.randn(B * T, d, generator=g) * 0.5).to(dev).bfloat16()
    ldp = (2 * T - 1 + 7) // 8 * 8
    dqkv = torch.zeros(B * T, 3 * d, device=dev, dtype=torch.bfloat16)
    vv = torch.empty(B * T, 3 * d, device=dev, dtype=torch.bfloat16)
    vv[:, 2 * d:] = v
    dS, dBD = ops.attn_fused_bwd(dctx, ctx, qu, vv[:, 2 * d:], p, pd, B, T, H, ldp, dqkv[:, d:2 * d], dqkv[:, 2 * d:], drop, 99)
    torch.cuda.synchronize()
    assert not dqkv[:, :d].any()  # the q slice is not touched
    dk_r = torch.empty(B * T, d, dtype=torch.bfloat16)
    dv_r = torch.empty(B * T, d, dtype=torch.bfloat16)
    dS_r, dBD_r = ops_ref.attn_fused_bwd(dctx.cpu(), ctx.cpu(), qu.cpu(), v.cpu(), p.cpu(), pd.cpu(), B, T, H, ldp, dk_r, dv_r,
                                         drop, 99)
    sc = max(dS_r.float().abs().max().item(), 1e-3)
    e_ds = (dS.float().cpu() - dS_r.float().cpu()).abs().max().item() / sc
    e_bd = (dBD.float().cpu() - dBD_r.float().cpu()).abs().max().item() / sc
    e_dk = (dqkv[:, d:2 * d].float().cpu() - dk_r.float().cpu()).abs().max().item() / max(dk_r.float().abs().max().item(), 1e-3)
    e_dv = (dqkv[:, 2 * d:].float().cpu() - dv_r.float().cpu()).abs().max().item() / max(dv_r.float().abs().max().item(), 1e-3)
    print("attn fused bwd B=%d T=%d H=%d drop=%.2f: dS %.2e dBD %.2e dK %.2e dV %.2e (max abs / max |ref|)" % (B, T, H, drop, e_ds, e_bd, e_dk, e_dv))
    # bf16 outputs; the row term comes from dctx.ctx (bf16 ctx) instead of sum_j P dP: a few bf16 ulps of the largest value
    assert e_ds < 2e-2 and e_bd < 2e-2 and e_dk < 2e-2 and e_dv < 2e-2, (e_ds, e_bd, e_dk, e_dv)
    # the skewed copy is exactly the plain one moved to columns (T-1)-i+j, zeros elsewhere
    i = torch.arange(T, device=dev)[:, None]
    j = torch.arange(T, device=dev)[None, :]
    idx = ((T - 1) - i + j).expand(H, B, T, T)
    assert torch.equal(dBD.gather(-1, idx), dS[..., :T])
    ref_sk = torch.zeros_like(dBD)
    ref_sk.scatter_(-1, idx, dS[..., :T])
    assert torch.equal(dBD, ref_sk)


@pytest.mark.parametrize("p,scale", [(0.0, 0.5), (0.1, 1.0), (0.3, 0.5)])
def test_layer_norm_bwd_second_output_is_the_next_dropout(dev, p, scale):
    """esp_layer_norm_bwd2: the extra output equals esp_dropout(dx, p, seed, scale) bit for bit (the next module's masked
    gradient comes out of the LayerNorm backward pass instead of a separate pass over dx)."""
    from espresso_b200 import ops

    R, d = 1000, 512
    g = torch.Generator(device="cpu").manual_seed(5)
    x = torch.randn(R, d, generator=g).to(dev).bfloat16()
    dy = torch.randn(R, d, generator=g).to(dev).bfloat16()
    dres = torch.randn(R, d, generator=g).to(dev).bfloat16()
    gamma = torch.randn(d, generator=g).to(dev).bfloat16()
    _, mean, rstd = ops.layer_norm_fwd(x, gamma, gamma, 1e-5)
    ga, gb = torch.zeros(d, device=dev), torch.zeros(d, device=dev)
    dx_ref = ops.layer_norm_bwd(dy, x, mean, rstd, gamma, ga, gb, dres=dres)
    ga2, gb2 = torch.zeros(d, device=dev), torch.zeros(d, device=dev)
    dx, dxd = ops.layer_norm_bwd(dy, x, mean, rstd, gamma, ga2, gb2, dres=dres, next_drop=(p, 777, scale))
    assert torch.equal(dx, dx_ref)
    assert torch.allclose(ga, ga2, rtol=1e-4, atol=1e-3) and torch.allclose(gb, gb2, rtol=1e-4, atol=1e-3)
    assert torch.equal(dxd, ops.dropout(dx_ref, p, 777, scale=scale))
