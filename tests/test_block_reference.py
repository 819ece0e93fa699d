"""CPU checks of the float64 block statements in oracle/block64.py, each against an independent result: float64 torch
autograd (F.layer_norm, F.glu + grouped F.conv1d, F.batch_norm + SiLU / ReLU, F.conv2d with one input channel), central
finite differences of the backward statements, the fp32 restatements of oracle/ops_ref.py (within a few fp32
roundings of the magnitude), and fairseq's recorded Adam trajectory in tests/golden/optimizer.npz."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import block64 as K
from oracle import ops_ref as O

F64, BF = torch.float64, torch.bfloat16


def _bf(shape, seed, scale=1.0, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=F64) * scale + shift).to(BF)


def _close(a, b, tol):
    a, b = a.to(F64), b.to(F64)
    assert float((a - b).abs().max()) <= tol * max(1.0, float(b.abs().max())), float((a - b).abs().max())


# ---------------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("R,d,shift", [(7, 8, 0.0), (9, 144, 0.0), (5, 520, 1000.0), (3, 1032, 0.0)])
def test_layer_norm_against_autograd(R, d, shift):
    x, gm, bt = _bf((R, d), 1, shift=shift), _bf(d, 2), _bf(d, 3)
    dy, dres = _bf((R, d), 4), _bf((R, d), 5)
    xr = x.to(F64).requires_grad_(True)
    gr, br = gm.to(F64).requires_grad_(True), bt.to(F64).requires_grad_(True)
    y = F.layer_norm(xr, (d,), gr, br, 1e-5)
    y.backward(dy.to(F64))
    f = K.layer_norm_fwd(x, gm, bt, 1e-5)
    _close(f.y, y.detach(), 1e-12)
    dg0, db0 = torch.randn(d, dtype=torch.float32), torch.randn(d, dtype=torch.float32)
    b = K.layer_norm_bwd(dy, x, f.mean, f.rstd, gm, dg0, db0, dres=dres)
    _close(b.dx, xr.grad + dres.to(F64), 1e-10)
    _close(b.dgamma, gr.grad + dg0.to(F64), 1e-10)
    _close(b.dbeta, br.grad + db0.to(F64), 1e-10)


def test_layer_norm_bwd_finite_differences():
    R, d = 3, 16
    x, gm, bt, dy = _bf((R, d), 6), _bf(d, 7), _bf(d, 8), _bf((R, d), 9)
    f = K.layer_norm_fwd(x, gm, bt, 1e-5)
    b = K.layer_norm_bwd(dy, x, f.mean, f.rstd, gm, torch.zeros(d), torch.zeros(d))
    xd, dyd = x.to(F64), dy.to(F64)

    def loss(xx):
        m = xx.mean(-1, keepdim=True)
        v = ((xx - m) ** 2).mean(-1, keepdim=True)
        return float((((xx - m) / torch.sqrt(v + 1e-5) * gm.to(F64) + bt.to(F64)) * dyd).sum())
    h = 1e-6
    fd = torch.zeros_like(xd)
    for i in range(R):
        for j in range(d):
            e = torch.zeros_like(xd)
            e[i, j] = h
            fd[i, j] = (loss(xd + e) - loss(xd - e)) / (2 * h)
    _close(b.dx, fd, 1e-6)


def test_layer_norm_lens_dropout_and_dx2_against_ops_ref():
    B, T, d = 3, 5, 64
    R = B * T
    x, gm, bt, dy = _bf((R, d), 10), _bf(d, 11), _bf(d, 12), _bf((R, d), 13)
    lens = torch.tensor([5, 0, 3], dtype=torch.int32)
    f = K.layer_norm_fwd(x, gm, bt, 1e-5, lens, T, 0.1, 77)
    y32, mean32, rstd32 = O.layer_norm_fwd(x, gm, bt, 1e-5, lens, T, 0.1, 77)
    assert K.tau_reached(y32, f.y, f.y_mag, bf16=True) < 8 * d * K.U32
    assert K.tau_reached(mean32, f.mean, f.mean_mag) < 4 * K.U32 * d
    assert K.tau_reached(rstd32, f.rstd, f.rstd_mag) < 4 * K.U32 * d
    dg, db = torch.zeros(d), torch.zeros(d)
    b = K.layer_norm_bwd(dy, x, mean32, rstd32, gm, dg.clone(), db.clone(), lens=lens, T=T, drop_p=0.1, seed=77,
                         next_drop=(0.1, 78, 0.5))
    dx32, dx2 = O.layer_norm_bwd(dy, x, mean32, rstd32, gm, dg, db, lens=lens, T=T, drop_p=0.1, seed=77,
                                 next_drop=(0.1, 78, 0.5))
    assert K.tau_reached(dx32, b.dx, b.dx_mag, bf16=True) < 8 * d * K.U32
    assert K.tau_reached(dg, b.dgamma, b.dgamma_mag) < 8 * R * K.U32
    assert torch.equal(b.dx2_of(dx32).view(torch.int16), dx2.view(torch.int16))
    assert (b.dx.view(B, T, d)[1] == 0).all() and (f.y.view(B, T, d)[2, 3:] == 0).all()


# ------------------------------------------------------------------------------------------------ GLU + depthwise conv
@pytest.mark.parametrize("B,T,C,k", [(2, 7, 8, 3), (1, 5, 16, 1), (2, 4, 8, 15), (1, 3, 8, 31)])
def test_glu_dwconv_against_autograd(B, T, C, k):
    g, w, dy = _bf((B, T, 2 * C), 14, 3.0), _bf((C, k), 15), _bf((B, T, C), 16)
    f = K.glu_dwconv_fwd(g, w)
    gl = f.glu.requires_grad_(True)  # the rounded GLU output feeds the conv
    wr = w.to(F64).requires_grad_(True)
    y = F.conv1d(gl.transpose(1, 2), wr[:, None, :], padding=k // 2, groups=C).transpose(1, 2)
    _close(f.y, y.detach(), 1e-12)
    y.backward(dy.to(F64))
    dw0 = torch.randn(C, k, dtype=torch.float32)
    b = K.glu_dwconv_bwd(dy, g, w, dw0)
    _close(b.dw, wr.grad + dw0.to(F64), 1e-12)
    gr = g.to(F64).requires_grad_(True)
    y2 = F.conv1d(F.glu(gr, -1).transpose(1, 2), w.to(F64)[:, None, :], padding=k // 2, groups=C).transpose(1, 2)
    y2.backward(dy.to(F64))
    _close(b.dg, gr.grad, 1e-12)
    st, _ = f.stats_of(K.rn(f.y))
    yb = K.rn(f.y).reshape(-1, C)
    _close(st, torch.stack([yb.sum(0), (yb * yb).sum(0)]), 1e-12)


def test_glu_dwconv_bwd_finite_differences():
    B, T, C, k = 1, 6, 8, 5
    g, w, dy = _bf((B, T, 2 * C), 17), _bf((C, k), 18), _bf((B, T, C), 19)
    b = K.glu_dwconv_bwd(dy, g, w, torch.zeros(C, k))
    gd, wd, dyd = g.to(F64), w.to(F64), dy.to(F64)

    def loss(gg):
        return float((K._dwconv(gg[..., :C] * torch.sigmoid(gg[..., C:]), wd) * dyd).sum())
    h = 1e-6
    fd = torch.zeros_like(gd)
    for t in range(T):
        for c in range(2 * C):
            e = torch.zeros_like(gd)
            e[0, t, c] = h
            fd[0, t, c] = (loss(gd + e) - loss(gd - e)) / (2 * h)
    _close(b.dg, fd, 1e-6)


def test_glu_dwconv_against_ops_ref():
    B, T, C, k = 2, 9, 16, 7
    g, w, dy = _bf((B, T, 2 * C), 20), _bf((C, k), 21), _bf((B, T, C), 22)
    f = K.glu_dwconv_fwd(g, w)
    y32, st32 = O.glu_dwconv_fwd(g, w)
    assert K.tau_reached(y32, f.y, f.y_mag, f.y_fl + f.y_mag * 2 ** -20, bf16=True) == 0
    dw32 = torch.zeros(C, k)
    dg32 = O.glu_dwconv_bwd(dy, g, w, dw32)
    b = K.glu_dwconv_bwd(dy, g, w, torch.zeros(C, k))
    assert K.tau_reached(dg32, b.dg, b.dg_mag, b.dg_fl, bf16=True) < 16 * K.U32 * k
    # ops_ref takes dw from the unrounded GLU output, the kernel (and block64) from the bf16 one: half a bf16 ulp apart
    assert 1e-4 < K.tau_reached(dw32, b.dw, b.dw_mag, b.dw_fl) < K.BF_REL


def test_rounded_flip_is_one_ulp_at_a_midpoint():
    x = torch.tensor([1.0 + 2 ** -8, 1.0 + 2 ** -9, 3.0], dtype=F64)  # a bf16 midpoint, an interior value, exact
    r, fl = K.rounded(x, torch.full_like(x, 1e-9))
    assert r.tolist() == [1.0, 1.0, 3.0] and fl.tolist() == [2 ** -7, 0.0, 0.0]


# ---------------------------------------------------------------------------------------------------------- BatchNorm
@pytest.mark.parametrize("act", [K.BN_ACT_SILU, K.BN_ACT_RELU])
@pytest.mark.parametrize("with_bias", [False, True])
def test_batchnorm_against_autograd(act, with_bias):
    R, C = 40, 16
    y, gm, bt, dz = _bf((R, C), 23, 2.0, 1.0), _bf(C, 24), _bf(C, 25), _bf((R, C), 26)
    pb = _bf(C, 27) if with_bias else None
    s = K.bn_stats(y, C, pb)
    rm, rv = torch.randn(C).abs(), torch.rand(C) + 0.5
    fin = K.bn_finalize(s.stats, R, C, 1e-5, 0.1, rm, rv, True)
    v, _ = K.pre(y, pb)
    rm_t, rv_t = rm.to(F64).clone(), rv.to(F64).clone()
    vr = v.clone().requires_grad_(True)
    gr, br = gm.to(F64).requires_grad_(True), bt.to(F64).requires_grad_(True)
    bn = F.batch_norm(vr, rm_t, rv_t, gr, br, training=True, momentum=0.1, eps=1e-5)
    _close(fin.run_mean, rm_t, 1e-12)
    _close(fin.run_var, rv_t, 1e-12)
    mr = torch.stack([fin.mean, fin.rstd])
    fw = K.bn_act_fwd(y, mr, gm, bt, act, pb)
    _close(fw.bn, K.rn(bn.detach()), 1e-12)
    want = F.silu(fw.bn) if act == K.BN_ACT_SILU else torch.relu(fw.bn)
    _close(fw.z, want, 1e-12)
    bw = K.bn_act_bwd(dz, y, mr, gm, bt, torch.zeros(C), torch.zeros(C), act, pb)
    ab = fw.bn.clone().requires_grad_(True)
    (F.silu(ab) if act == K.BN_ACT_SILU else torch.relu(ab)).backward(dz.to(F64))
    bn.backward(ab.grad)  # the BatchNorm backward of dbn = dz act'(RN(bn))
    _close(bw.dy, vr.grad, 1e-10)
    _close(bw.dgamma, gr.grad, 1e-10)
    _close(bw.dbeta, br.grad, 1e-10)


def test_batchnorm_bwd_finite_differences():
    R, C = 12, 8
    y, gm, bt, dz = _bf((R, C), 28), _bf(C, 29), _bf(C, 30), _bf((R, C), 31)
    s = K.bn_stats(y, C)
    fin = K.bn_finalize(s.stats, R, C, 1e-5, 0.1, None, None, True)
    mr = torch.stack([fin.mean, fin.rstd])
    dbn = dz.to(F64)  # identity activation: the BatchNorm backward alone, through act' = 1 for bn > 0 ...
    bw = K.bn_act_bwd(dz, y, mr, gm, bt.to(F64).add(100.0).to(BF), torch.zeros(C), torch.zeros(C), K.BN_ACT_RELU)
    yd = y.to(F64)

    def loss(yy):
        m = yy.mean(0)
        rs = 1 / torch.sqrt(((yy - m) ** 2).mean(0) + 1e-5)
        return float(((yy - m) * rs * gm.to(F64) * dbn).sum())  # ... shifted by beta + 100 so that every bn > 0
    h = 1e-6
    fd = torch.zeros_like(yd)
    for i in range(R):
        for j in range(C):
            e = torch.zeros_like(yd)
            e[i, j] = h
            fd[i, j] = (loss(yd + e) - loss(yd - e)) / (2 * h)
    _close(bw.dy, fd, 1e-6)


def test_batchnorm_against_ops_ref_and_eval():
    R, C = 64, 32
    y, gm, bt, dz, pb = _bf((R, C), 32, 3.0), _bf(C, 33), _bf(C, 34), _bf((R, C), 35), _bf(C, 36)
    s = K.bn_stats(y, C, pb)
    assert K.tau_reached(O.bn_stats(y, C, pb), s.stats, s.stats_mag, s.stats_fl) < 1e-12
    rm, rv = torch.randn(C), torch.rand(C) + 0.5
    mr32 = O.bn_finalize(O.bn_stats(y, C, pb), R, C, 1e-5, 0.1, rm.clone(), rv.clone(), True)
    fin = K.bn_finalize(s.stats, R, C, 1e-5, 0.1, rm, rv, True)
    assert K.tau_reached(mr32[1], fin.rstd, fin.rstd_mag) < 8 * K.U32
    ev = K.bn_finalize(None, 0, C, 1e-5, 0.1, rm, rv, False)
    assert torch.equal(ev.mean, rm.to(F64)) and K.tau_reached(1 / torch.sqrt(rv.to(F64) + 1e-5), ev.rstd, ev.rstd_mag) < 1e-15
    for act in (K.BN_ACT_SILU, K.BN_ACT_RELU):
        fw = K.bn_act_fwd(y, mr32, gm, bt, act, pb)
        assert K.tau_reached(O.bn_act_fwd(y, mr32, gm, bt, act, pb), fw.z, fw.z_mag, fw.z_fl + 1e-6 * fw.bn.abs(), True) == 0
        dg, db = torch.zeros(C), torch.zeros(C)
        dy32 = O.bn_act_bwd(dz, y, mr32, gm, bt, dg, db, act, pb)
        bw = K.bn_act_bwd(dz, y, mr32, gm, bt, torch.zeros(C), torch.zeros(C), act, pb)
        assert K.tau_reached(dy32, bw.dy, bw.dy_mag, bw.dy_fl, True) < 16 * R * K.U32
        assert K.tau_reached(dg, bw.dgamma, bw.dgamma_mag, bw.dgamma_fl) < 16 * R * K.U32


# ---------------------------------------------------------------------------------------------- first conv (Cin = 1)
@pytest.mark.parametrize("T,Fb,stride", [(5, 7, (1, 1)), (6, 9, (2, 2)), (7, 5, (3, 1)), (1, 1, (2, 2))])
def test_conv3x3_c1_against_autograd(T, Fb, stride):
    B, Cout = 2, 8
    x, w = _bf((B, T, Fb), 37), _bf((Cout, 3, 3), 38)
    xr, wr = x.to(F64)[:, None].requires_grad_(True), w.to(F64)[:, None].requires_grad_(True)
    y = F.conv2d(xr, wr, None, stride, 1)
    y64, mag = K.conv3x3_c1_fwd(x, w, stride)
    _close(y64, y.detach().permute(0, 2, 3, 1), 1e-12)
    assert (mag >= y64.abs()).all()
    dy = _bf(y64.shape, 39)
    y.backward(dy.to(F64).permute(0, 3, 1, 2))
    dw0 = torch.randn(Cout, 3, 3)
    dw, _ = K.conv3x3_c1_wgrad(dy, x, stride, dw0)
    _close(dw, wr.grad[:, 0] + dw0.to(F64), 1e-12)


# -------------------------------------------------------------------------------------------------------------- optimizer
def test_adam_statement_replays_fairseq_trajectory(golden_dir):
    g = np.load(os.path.join(golden_dir, "optimizer.npz"))
    lr, b1, b2, eps, wd, clip = g["hyper"].tolist()
    p = torch.from_numpy(g["p0"]).to(F64)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    for step in range(1, 5):
        grad = torch.from_numpy(g["g%d" % step]).to(F64)
        r = K.adam_step(p, m, v, grad, lr, b1, b2, eps, wd, step, float((grad * grad).sum()), float(g["ss%d" % step]), clip)
        assert abs(r.gnorm - float(g["gnorm%d" % step])) <= 1e-6 * float(g["gnorm%d" % step])
        # the recording is fp32: one fp32 rounding per operation of the step
        assert float(((r.p - torch.from_numpy(g["p%d" % step]).to(F64)).abs() / r.p_mag).max()) < 64 * K.U32
        p, m, v = torch.from_numpy(g["p%d" % step]).to(F64), r.m, r.v


def test_adam_against_ops_ref_and_pow_err():
    n = 1000
    gen = torch.Generator().manual_seed(40)
    p, m, v = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 1e-2, torch.rand(n, generator=gen) * 1e-4
    grad = torch.randn(n, generator=gen) * 3
    for step, beta2, wd, clip in [(1, 0.98, 0.0, 0.0), (10, 0.999, 0.01, 1.0), (100000, 0.98, 0.01, 1e6)]:
        ss = float((grad.double() ** 2).sum())
        r = K.adam_step(p, m, v, grad, 1e-3, 0.9, beta2, 1e-8, wd, step, ss, 4.0, clip)
        p32, m32, v32 = p.clone(), m.clone(), v.clone()
        O.adam_step(p32, m32, v32, grad, p32.to(BF), 1e-3, 0.9, beta2, 1e-8, wd, step, torch.tensor([ss]),
                    denom_const=4.0, clip_norm=clip)
        # ops_ref scales by the double 1 - beta (as fairseq's fp32 tensor ops do), the statement by 1 - fp32(beta), the
        # kernel's own input: they differ by that coefficient's relative change
        tol = 16 * K.U32 + 2 * max(abs((1 - float(np.float32(bb))) / (1 - bb) - 1) for bb in (0.9, beta2))
        assert K.tau_reached(p32, r.p, r.p_mag, r.p_fl) < tol
        assert K.tau_reached(m32, r.m, r.m_mag) < tol and K.tau_reached(v32, r.v, r.v_mag) < tol
    # pow_err covers fp32 betas raised to large steps: 1 - powf(fp32(0.999), s) against 1 - 0.999^s
    for s in (1, 10, 1000, 100000):
        got = 1 - float(np.float32(np.power(np.float32(0.999), np.float32(s), dtype=np.float32)))
        assert abs(got - (1 - 0.999 ** s)) <= K.pow_err(0.999, s)
