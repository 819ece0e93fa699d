"""The block kernels of csrc/elementwise.cu and csrc/optim.cu against the float64 statements of oracle/block64.py, per
element, on every kernel branch: LayerNorm forward / backward (all three NV instances, the vector and the atomicAdd
parameter-gradient paths, the fused dx2), column sums, q preparation, row masking, GLU + depthwise conv (+ statistics),
BatchNorm statistics / finalize / activation forward and backward (SiLU and ReLU, with and without pre_bias), the
one-input-channel first convolution, and the optimizer (squared norm, fused clip + Adam, casts).  Outputs sit between
NaN-payload sentinels; every case writes the error it reached next to its bound through the `parity` fixture.

Bounds: per element, |x - x64| <= tau * mag + fl for fp32 outputs and 2^-8 |x64| + (1 + 2^-8)(tau * mag + fl) for bf16
outputs, with mag and fl from oracle/block64.py.  Each tau below is about 2x the largest value reached on an NVIDIA H100
80GB HBM3 (700 W power limit); a tau whose reached value is 0 (the bf16 rounding and flip terms cover every element)
keeps its analytic value, marked "analytic".  A dropped bf16 rounding point, a tap off by one, a missing t < T guard, a
scratch slot left non-zero or a skipped atomicAdd path moves some element by far more than its bound."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import block64 as K

pytestmark = pytest.mark.gpu

BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
TAU_LN = 8e-8  # LayerNorm y, dx per unit of magnitude: reached 3.9e-8 (y, d = 2048)
TAU_LN_STAT = 8e-7  # LayerNorm mean (per mean|x|) and rstd (relative): reached 4.0e-7 (rstd, rows of 1000 + N(0,1))
TAU_LN_PARAM = 5e-7  # dgamma / dbeta over up to 6600 rows: reached 2.5e-7
TAU_COLSUM = 2.2e-7  # column sums over up to 20000 rows: reached 1.1e-7
TAU_DW = 4e-8  # GLU + dwconv y, dg: reached 1.8e-8 (C = 1024, k = 31)
TAU_DW_PARAM = 2.2e-7  # dw and the dwconv statistics: reached 1.1e-7
TAU_BN_STATS = 7e-7  # bn_stats and the bn_act_bwd sums: reached 3.5e-7 (C = 8), 2.5e-7 at 2.1 M rows
TAU_BN = 1e-8  # bn_act_bwd dy: reached 3.0e-9
TAU_BN_Z = 2 * K.U32  # bn_act z: reached 0 (bf16 rounding and flips cover every element), analytic
TAU_FIN = 4 * K.U32  # bn_finalize mean, rstd, running statistics: reached 1.1e-7
TAU_C1 = 6e-9  # conv3x3_c1 forward (9 exact products per output): reached 2.7e-9
TAU_C1_W = 2.3e-7  # conv3x3_c1 wgrad: reached 1.1e-7
TAU_SUMSQ = 1.5e-6  # sumsq up to 3e7 elements: reached 6.4e-7 (n = 3e7; the float atomics' order varies)
TAU_ADAM = 8e-7  # Adam p, m, v and gnorm: reached 3.6e-7 (v), 1.1e-7 (p, gnorm)
GRAD_REL = 1.25e-2    # compositions: ||g - g64|| / ||g64|| of every output and gradient
GRAD_REL_FRONT = 4e-2  # the first conv's dw, dgamma, dbeta against float64 end to end: reached 2.2e-2 (see the test)
SENT16 = 0x7FA5
SENT32 = 0x7FC0DEAD
SENT64 = 0x7FF8DEADBEEF0001


@pytest.fixture(scope="module", autouse=True)
def _env():
    from espresso_b200 import ops

    assert torch.cuda.is_available()
    saved = ops._SEED_T
    ops.set_seed_tensor(None)
    yield
    ops.set_seed_tensor(saved)


def _lib():
    from espresso_b200 import lib

    return lib


def _L():
    return _lib().load()


def _ops():
    from espresso_b200 import ops

    return ops


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rand(shape, seed, scale=1.0, shift=0.0):
    return (torch.randn(shape, generator=_gen(seed), device="cuda", dtype=F32) * scale + shift).to(BF)


_IV = {BF: (torch.int16, SENT16), F32: (torch.int32, SENT32), F64: (torch.int64, SENT64)}


def _boxed(shape, dtype=BF, pad=64, off=0, init=None):
    """A tensor of `shape` inside a flat sentinel buffer (pad sentinels either side, `off` more elements before the
    view) -> (buffer, view); init fills the view."""
    n = int(np.prod(shape)) if len(shape) else 1
    it, s = _IV[dtype]
    buf = torch.empty(n + 2 * pad + off, device="cuda", dtype=dtype)
    buf.view(it).fill_(s)
    view = buf[pad + off:pad + off + n].view(shape)
    if init is not None:
        view.copy_(init)
    return buf, view


def _untouched(buf, view, what):
    flat = buf.reshape(-1)
    mark = torch.zeros(flat.numel(), dtype=torch.bool, device=buf.device)
    idx = torch.arange(flat.numel(), device=buf.device)
    mark[idx.as_strided(view.shape, view.stride(), view.storage_offset() - buf.storage_offset()).reshape(-1)] = True
    it, s = _IV[buf.dtype]
    bad = (~mark) & (flat.view(it) != s)
    assert not bad.any(), "%s: %d elements written outside the output" % (what, int(bad.sum()))


def _check(parity, name, got, val, mag, tau, fl=0.0, bf16=False):
    assert not torch.isnan(got).any(), name + ": NaN"
    parity(name, K.tau_reached(got, val, mag, fl, bf16), tau)


def _rel(parity, name, got, ref, bound=GRAD_REL):
    parity(name, float((got.to(F64) - ref).norm() / ref.norm().clamp_min(1e-300)), bound)


# ---------------------------------------------------------------------------------------------------------- LayerNorm
LN_D = [8, 144, 256, 512, 520, 768, 1024, 1032, 2048]
LN_R = [1, 7, 8, 9, 24 * 275]


def _ln_lens(R):
    """Ragged [B, T] rows with a 0 and a full length; None for R = 1 (lens = [1] is the T = R = 1 case below)."""
    B, T = {1: (1, 1), 7: (1, 7), 8: (2, 4), 9: (3, 3), 24 * 275: (24, 275)}.get(R, (R // 25, 25))
    vals = [T] + [(T * (b + 1)) // (B + 1) for b in range(1, B)]
    if B > 1:
        vals[1] = 0
    return torch.tensor(vals, dtype=torch.int32, device="cuda"), T


def _ln_x(R, d, kind, seed):
    if kind == "randn":
        return _rand((R, d), seed)
    if kind == "mean1000":
        return _rand((R, d), seed, 1.0, 1000.0)
    row = _rand((R, 1), seed, 3.0)  # constant rows: variance 0, rstd = 1/sqrt(eps)
    return row.expand(R, d).contiguous()


def _ln_case(parity, d, R, kind="randn", lens=True, dres=True, misaligned=False, drop_p=0.0, p2=0.1, scale2=0.5):
    tag = "ln d=%d R=%d %s lens=%d dres=%d mis=%d p=%g p2=%g" % (d, R, kind, lens, dres, misaligned, drop_p, p2)
    x = _ln_x(R, d, kind, d + R)
    gm, bt = _rand(d, 1, 0.5, 1.0), _rand(d, 2, 0.3)
    ln, T = _ln_lens(R) if lens else (None, 0)
    yb, y = _boxed((R, d))
    mb, mean = _boxed((R,), F32)
    rb, rstd = _boxed((R,), F32)
    seed = 1000 + d
    assert _L().esp_layer_norm_fwd(_p(x), _p(gm), _p(bt), 1e-5, R, d, _p(y), _p(mean), _p(rstd), _p(ln), T, drop_p, seed,
                                   None, _stream()) == 0
    f = K.layer_norm_fwd(x, gm, bt, 1e-5, ln, T, drop_p, seed)
    torch.cuda.synchronize()
    for b, v, w in ((yb, y, "y"), (mb, mean, "mean"), (rb, rstd, "rstd")):
        _untouched(b, v, tag + " " + w)
    _check(parity, tag + " y", y, f.y, f.y_mag, TAU_LN, bf16=True)
    _check(parity, tag + " mean", mean, f.mean, f.mean_mag, TAU_LN_STAT)
    _check(parity, tag + " rstd", rstd, f.rstd, f.rstd_mag, TAU_LN_STAT)
    # backward from the kernel's own mean / rstd, accumulating onto non-zero parameter gradients
    dy = _rand((R, d), seed + 1)
    dr = _rand((R, d), seed + 2) if dres else None
    dg0 = torch.randn(d, generator=_gen(seed + 3), device="cuda")
    db0 = torch.randn(d, generator=_gen(seed + 4), device="cuda")
    off = 1 if misaligned else 0
    dgb, dg = _boxed((d,), F32, off=off, init=dg0)
    dbb, db = _boxed((d,), F32, off=off, init=db0)
    dxb, dx = _boxed((R, d))
    d2b, dx2 = _boxed((R, d))
    assert _L().esp_layer_norm_bwd2(_p(dy), _p(x), _p(mean), _p(rstd), _p(gm), _p(dr), R, d, _p(dx), _p(dg), _p(db), _p(ln), T,
                                    drop_p, seed, None, _p(dx2), p2, seed + 5, scale2, _stream()) == 0
    b = K.layer_norm_bwd(dy, x, mean, rstd, gm, dg0, db0, dr, ln, T, drop_p, seed, next_drop=(p2, seed + 5, scale2))
    torch.cuda.synchronize()
    for bb, v, w in ((dgb, dg, "dgamma"), (dbb, db, "dbeta"), (dxb, dx, "dx"), (d2b, dx2, "dx2")):
        _untouched(bb, v, tag + " " + w)
    _check(parity, tag + " dx", dx, b.dx, b.dx_mag, TAU_LN, bf16=True)
    _check(parity, tag + " dgamma", dg, b.dgamma, b.dgamma_mag, TAU_LN_PARAM)
    _check(parity, tag + " dbeta", db, b.dbeta, b.dbeta_mag, TAU_LN_PARAM)
    want = b.dx2_of(dx)
    assert torch.equal(dx2.view(torch.int16), want.view(torch.int16)), tag + ": dx2 is not dropout(bf16(dx)) * scale2"
    parity(tag + " dx2 bit-exact", 0.0, 0.0)


@pytest.mark.parametrize("R", LN_R)
@pytest.mark.parametrize("d", LN_D)
def test_layer_norm_every_instance(parity, d, R):
    _ln_case(parity, d, R, p2=0.1 if R < 100 or d == 512 else 0.0)


@pytest.mark.parametrize("d", [144, 512, 1032, 2048])
@pytest.mark.parametrize("kind", ["mean1000", "const"])
def test_layer_norm_large_mean_and_constant_rows(parity, d, kind):
    _ln_case(parity, d, 9, kind, lens=False, dres=False, p2=0.0, scale2=2.0)
    _ln_case(parity, d, 600, kind)


@pytest.mark.parametrize("d", [144, 520, 1032])
def test_layer_norm_misaligned_param_grads(parity, d):
    """dgamma / dbeta views one float off 16-byte alignment: the atomicAdd path."""
    _ln_case(parity, d, 600, misaligned=True)
    _ln_case(parity, d, 7, misaligned=True, dres=False, lens=False)


@pytest.mark.parametrize("d", [256, 1024])
def test_layer_norm_dropout(parity, d):
    _ln_case(parity, d, 9, drop_p=0.1, p2=0.1, scale2=0.75)
    _ln_case(parity, d, 300, drop_p=0.1, p2=0.0, scale2=0.75, lens=False)


# --------------------------------------------------------------------------------------------------------- column sums
@pytest.mark.parametrize("R", [1, 33, 20000])
@pytest.mark.parametrize("N", [8, 264, 4096, 4104, 8200])
def test_colsum(parity, N, R):
    ld = N + 24
    out0 = torch.randn(N, generator=_gen(N), device="cuda")
    ob, out = _boxed((N,), F32, init=out0)
    exp, mag = out0.to(F64), out0.to(F64).abs()
    for call in range(2):  # the second call proves the scratch slots and tickets were reset by the first
        xb, xs = _boxed((R, ld), init=_rand((R, ld), N + R + call, 2.0))
        x = xs[:, :N]
        assert _L().esp_colsum(_p(x), R, N, ld, 0.37, _p(out), _stream()) == 0
        r = K.colsum(x, torch.zeros(N, device="cuda"), 0.37)
        exp, mag = exp + r.out, mag + r.out_mag
        torch.cuda.synchronize()
        _untouched(ob, out, "colsum out")
        _check(parity, "colsum N=%d R=%d call %d" % (N, R, call), out, exp, mag, TAU_COLSUM)


# ---------------------------------------------------------------------------------------------- q prep and row masks
@pytest.mark.parametrize("R,d", [(1, 8), (37, 64), (600, 512)])
def test_qprep_exact(parity, R, d):
    ldq = 3 * d
    qfull = _rand((R, ldq), R + d, 3.0)
    q = qfull[:, d:2 * d]
    u, v = _rand(d, 5, 0.5), _rand(d, 6, 0.5)
    qub, qu = _boxed((R, d))
    qvb, qv = _boxed((R, d))
    s = 0.125 * 1.1
    assert _L().esp_qprep_fwd(_p(q), ldq, _p(u), _p(v), s, R, d, _p(qu), _p(qv), _stream()) == 0
    equ, eqv = K.qprep_fwd(q, u, v, s)
    dqu, dqv = _rand((R, d), 7), _rand((R, d), 8)
    dqb, dqfull = _boxed((R, ldq))
    dq = dqfull[:, :d]
    assert _L().esp_qprep_bwd(_p(dqu), _p(dqv), s, R, d, _p(dq), ldq, _stream()) == 0
    torch.cuda.synchronize()
    _untouched(qub, qu, "qu")
    _untouched(qvb, qv, "qv")
    _untouched(dqb, dq, "dq (strided rows)")
    assert torch.equal(qu.view(torch.int16), equ.view(torch.int16))
    assert torch.equal(qv.view(torch.int16), eqv.view(torch.int16))
    assert torch.equal(dq.contiguous().view(torch.int16), K.qprep_bwd(dqu, dqv, s).view(torch.int16))
    parity("qprep R=%d d=%d bit-exact" % (R, d), 0.0, 0.0)


def test_mask_rows_exact(parity):
    B, T, N = 4, 37, 136
    x = _rand((B, T, N), 9)
    lens = torch.tensor([37, 0, 1, 20], dtype=torch.int32, device="cuda")
    xb, xv = _boxed((B, T, N), init=x)
    assert _L().esp_mask_rows(_p(xv), _p(lens), B, T, N, _stream()) == 0
    torch.cuda.synchronize()
    _untouched(xb, xv, "mask_rows")
    assert torch.equal(xv.view(torch.int16), K.mask_rows(x, lens).view(torch.int16))
    parity("mask_rows bit-exact", 0.0, 0.0)


# ------------------------------------------------------------------------------------------------ GLU + depthwise conv
def _glu_input(B, T, C, seed, gates=None):
    a = _rand((B, T, C), seed, 1.0)
    gate = _rand((B, T, C), seed + 1, 2.0)
    if gates is not None:  # saturated gates on a quarter of the elements
        sel = torch.rand((B, T, C), generator=_gen(seed + 2), device="cuda") < 0.25
        pick = torch.randint(0, len(gates), (B, T, C), generator=_gen(seed + 3), device="cuda")
        gate = torch.where(sel, torch.tensor(gates, device="cuda", dtype=F32)[pick].to(BF), gate)
    return torch.cat([a, gate], -1).contiguous()


def _dwconv_case(parity, B, T, C, k, gates=None, seed=0):
    tag = "dwconv B=%d T=%d C=%d k=%d%s" % (B, T, C, k, " saturated" if gates else "")
    g = _glu_input(B, T, C, 100 + seed + k + T, gates)
    w = _rand((C, k), 200 + k, 0.3)
    s0 = torch.randn(2, C, generator=_gen(5), device="cuda", dtype=F64)
    yb, y = _boxed((B, T, C))
    sb, st = _boxed((2, C), F64, init=s0)
    assert _L().esp_glu_dwconv_fwd(_p(g), _p(w), B, T, C, k, _p(y), _p(st), _stream()) == 0
    f = K.glu_dwconv_fwd(g, w)
    torch.cuda.synchronize()
    _untouched(yb, y, tag + " y")
    _untouched(sb, st, tag + " stats")
    _check(parity, tag + " y", y, f.y, f.y_mag, TAU_DW, f.y_fl, bf16=True)
    sv, sm = f.stats_of(y)
    _check(parity, tag + " stats", st, s0 + sv, s0.abs() + sm, TAU_DW_PARAM)
    dy = _rand((B, T, C), 300 + k + T)
    dw0 = torch.randn(C, k, generator=_gen(6), device="cuda")
    gb, dg = _boxed((B, T, 2 * C))
    wb, dw = _boxed((C, k), F32, init=dw0)
    assert _L().esp_glu_dwconv_bwd(_p(dy), _p(g), _p(w), B, T, C, k, _p(dg), _p(dw), _stream()) == 0
    b = K.glu_dwconv_bwd(dy, g, w, dw0)
    torch.cuda.synchronize()
    _untouched(gb, dg, tag + " dg")
    _untouched(wb, dw, tag + " dw")
    _check(parity, tag + " dg", dg, b.dg, b.dg_mag, TAU_DW, b.dg_fl, bf16=True)
    _check(parity, tag + " dw", dw, b.dw, b.dw_mag, TAU_DW_PARAM, b.dw_fl)
    assert not torch.isnan(y).any() and not torch.isnan(dg).any()


@pytest.mark.parametrize("T", [1, 2, 15, 63, 64, 65, 275])
@pytest.mark.parametrize("k", [1, 3, 15, 31])
def test_glu_dwconv_taps_and_tiles(parity, k, T):
    _dwconv_case(parity, 3, T, 64, k)


@pytest.mark.parametrize("B,T,C", [(1, 275, 512), (24, 65, 512), (1, 130, 1024), (24, 275, 1024)])
def test_glu_dwconv_channels_and_batch(parity, B, T, C):
    _dwconv_case(parity, B, T, C, 31)


@pytest.mark.parametrize("k", [3, 31])
def test_glu_dwconv_saturated_gates(parity, k):
    _dwconv_case(parity, 2, 70, 128, k, gates=[90.0, -90.0, 1e4, -1e4], seed=7)


# ---------------------------------------------------------------------------------------------------------- BatchNorm
BN_C = [8, 16, 32, 64, 128, 256, 512, 1024, 2048]


def _bn_stats_case(parity, tag, x, C_, pb):
    R = x.numel() // C_
    s0 = torch.randn(2, C_, generator=_gen(C_), device="cuda", dtype=F64)
    sb, st = _boxed((2, C_), F64, init=s0)
    assert _L().esp_bn_stats(_p(x), _p(pb), R, C_, _p(st), _stream()) == 0
    r = K.bn_stats(x, C_, pb)
    torch.cuda.synchronize()
    _untouched(sb, st, tag)
    _check(parity, tag, st, s0 + r.stats, s0.abs() + r.stats_mag, TAU_BN_STATS, r.stats_fl)
    return st - s0


@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("C_", BN_C)
def test_bn_stats_every_channel_count(parity, C_, with_bias):
    R = 4099
    x = _rand((R, C_), C_, 2.0, 0.5)
    pb = _rand(C_, C_ + 1, 0.7) if with_bias else None
    _bn_stats_case(parity, "bn_stats C=%d R=%d bias=%d" % (C_, R, with_bias), x, C_, pb)


def test_bn_stats_mean_std_10(parity):
    x = _rand((50000, 64), 11, 10.0, 10.0)
    _bn_stats_case(parity, "bn_stats mean/std 10", x, 64, _rand(64, 12, 0.5))


def test_bn_front_recipe_size(parity):
    """The conv front's first BatchNorm: B = 24, T = 1100, F = 80, C = 64 (2.1 M rows), mean / std 10, with pre_bias:
    statistics, finalize and the backward's two sums at full size."""
    B, T, Fb, C_ = 24, 1100, 80, 64
    R = B * T * Fb
    x = _rand((R, C_), 13, 10.0, 10.0)
    pb = _rand(C_, 14, 0.5)
    st = _bn_stats_case(parity, "bn_stats recipe 2.1M rows", x, C_, pb)
    mr = _ops().bn_finalize(st.contiguous(), R, C_, 1e-5, 0.1, None, None, True)
    _bn_act_case(parity, "bn_act recipe 2.1M rows", x, mr, C_, K.BN_ACT_RELU, pb, seed=15)


def _bn_finalize_case(parity, tag, st, R, C_, training):
    rm0 = torch.randn(C_, generator=_gen(16), device="cuda")
    rv0 = torch.rand(C_, generator=_gen(17), device="cuda") + 0.5
    rmb, rm = _boxed((C_,), F32, init=rm0)
    rvb, rv = _boxed((C_,), F32, init=rv0)
    mrb, mr = _boxed((2, C_), F32)
    assert _L().esp_bn_finalize(_p(st), R, C_, 1e-5, 0.1, _p(rm), _p(rv), int(training), _p(mr), _stream()) == 0
    r = K.bn_finalize(st, R, C_, 1e-5, 0.1, rm0, rv0, training)
    torch.cuda.synchronize()
    for b, v, w in ((rmb, rm, "run_mean"), (rvb, rv, "run_var"), (mrb, mr, "mr")):
        _untouched(b, v, tag + " " + w)
    _check(parity, tag + " mean", mr[0], r.mean, r.mean_mag, TAU_FIN)
    _check(parity, tag + " rstd", mr[1], r.rstd, r.rstd_mag, TAU_FIN)
    if training:
        _check(parity, tag + " running mean", rm, r.run_mean, r.run_mean_mag, TAU_FIN)
        _check(parity, tag + " running var", rv, r.run_var, r.run_var_mag, TAU_FIN)
    else:
        assert torch.equal(rm, rm0) and torch.equal(rv, rv0)


@pytest.mark.parametrize("R", [1, 2, 4099])
@pytest.mark.parametrize("training", [True, False])
def test_bn_finalize(parity, R, training):
    C_ = 64
    x = _rand((R, C_), 18 + R, 3.0, 1.0).to(F64)
    st = torch.stack([x.sum(0), (x * x).sum(0)]).contiguous()
    _bn_finalize_case(parity, "bn_finalize R=%d training=%d" % (R, training), st, R, C_, training)


def _bn_act_case(parity, tag, y, mr, C_, act, pb, seed, zeros=None):
    R = y.numel() // C_
    gm, bt = _rand(C_, seed, 0.5, 1.0), _rand(C_, seed + 1, 0.3)
    if zeros is not None:
        bt = torch.where(zeros, torch.zeros_like(bt), bt)
    zb, z = _boxed((R, C_))
    assert _L().esp_bn_act_fwd(_p(y), _p(pb), R, C_, _p(mr), _p(gm), _p(bt), act, _p(z), _stream()) == 0
    f = K.bn_act_fwd(y, mr, gm, bt, act, pb)
    torch.cuda.synchronize()
    _untouched(zb, z, tag + " z")
    _check(parity, tag + " z", z, f.z, f.z_mag, TAU_BN_Z, f.z_fl, bf16=True)
    dz = _rand((R, C_), seed + 2)
    dg0 = torch.randn(C_, generator=_gen(seed + 3), device="cuda")
    db0 = torch.randn(C_, generator=_gen(seed + 4), device="cuda")
    dgb, dg = _boxed((C_,), F32, init=dg0)
    dbb, db = _boxed((C_,), F32, init=db0)
    wsb, ws = _boxed((3, C_), F64)
    dyb, dy = _boxed((R, C_))
    assert _L().esp_bn_act_bwd(_p(dz), _p(y), _p(pb), R, C_, _p(mr), _p(gm), _p(bt), act, _p(ws), _p(dy), _p(dg), _p(db),
                               _stream()) == 0
    b = K.bn_act_bwd(dz, y, mr, gm, bt, dg0, db0, act, pb)
    torch.cuda.synchronize()
    for bb, v, w in ((dgb, dg, "dgamma"), (dbb, db, "dbeta"), (wsb, ws, "workspace"), (dyb, dy, "dy")):
        _untouched(bb, v, tag + " " + w)
    _check(parity, tag + " dy", dy, b.dy, b.dy_mag, TAU_BN, b.dy_fl, bf16=True)
    _check(parity, tag + " dgamma", dg, b.dgamma, b.dgamma_mag, TAU_BN_STATS, b.dgamma_fl)
    _check(parity, tag + " dbeta", db, b.dbeta, b.dbeta_mag, TAU_BN_STATS, b.dbeta_fl)
    return f, b


@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("act", [1, 2])
@pytest.mark.parametrize("C_", [8, 64, 512, 2048])
def test_bn_act(parity, C_, act, with_bias):
    R = 3001
    y = _rand((R, C_), 20 + C_, 2.0, 0.5)
    pb = _rand(C_, 21, 0.7) if with_bias else None
    v, _ = K.pre(y, pb)
    v = v.reshape(R, C_)
    mean, var = v.mean(0), v.var(0, unbiased=False)
    mr = torch.stack([mean, 1 / torch.sqrt(var + 1e-5)]).to(F32).contiguous()
    _bn_act_case(parity, "bn_act C=%d act=%d bias=%d" % (C_, act, with_bias), y, mr, C_, act, pb, seed=22)


@pytest.mark.parametrize("act", [1, 2])
def test_bn_act_exact_zero_outputs(parity, act):
    """bn == 0 exactly on half of the channels of every other row: ReLU' there is 0 (strict), and SiLU(0) = 0."""
    R, C_ = 512, 64
    mean = _rand(C_, 23, 1.0)
    y = _rand((R, C_), 24, 2.0)
    zero_c = torch.arange(C_, device="cuda") % 2 == 0
    hit = (torch.arange(R, device="cuda")[:, None] % 2 == 0) & zero_c[None, :]
    y = torch.where(hit, mean.expand(R, C_), y).contiguous()
    mr = torch.stack([mean.float(), torch.full((C_,), 0.75, device="cuda")]).contiguous()
    f, _ = _bn_act_case(parity, "bn_act exact zeros act=%d" % act, y, mr, C_, act, None, seed=25, zeros=zero_c)
    assert bool((f.bn.reshape(R, C_)[hit] == 0).all())


# ---------------------------------------------------------------------------------------------- first conv (Cin = 1)
def _c1_case(parity, B, T, Fb, Cout, st, sf, seed):
    tag = "conv3x3_c1 B=%d T=%d F=%d Cout=%d st=%d sf=%d" % (B, T, Fb, Cout, st, sf)
    x = _rand((B, T, Fb), seed, 1.5)
    w = _rand((Cout, 3, 3), seed + 1, 0.5)
    To, Fo = (T + st - 1) // st, (Fb + sf - 1) // sf
    yb, y = _boxed((B, To, Fo, Cout))
    assert _L().esp_conv3x3_c1_fwd(_p(x), _p(w), _p(y), B, T, Fb, Cout, st, sf, _stream()) == 0
    y64, mag = K.conv3x3_c1_fwd(x, w, (st, sf))
    dy = _rand((B, To, Fo, Cout), seed + 2)
    dw0 = torch.randn(Cout, 3, 3, generator=_gen(seed + 3), device="cuda")
    wb, dw = _boxed((Cout, 3, 3), F32, init=dw0)
    assert _L().esp_conv3x3_c1_wgrad(_p(dy), _p(x), _p(dw), B, T, Fb, Cout, st, sf, _stream()) == 0
    dw64, dmag = K.conv3x3_c1_wgrad(dy, x, (st, sf), dw0)
    torch.cuda.synchronize()
    _untouched(yb, y, tag + " y")
    _untouched(wb, dw, tag + " dw")
    _check(parity, tag + " y", y, y64, mag, TAU_C1, bf16=True)
    _check(parity, tag + " dw", dw, dw64, dmag, TAU_C1_W)


@pytest.mark.parametrize("sf", [1, 2])
@pytest.mark.parametrize("st", [1, 2, 3])
@pytest.mark.parametrize("Fb", [1, 2, 3, 5, 80, 83])
def test_conv3x3_c1_strides_and_widths(parity, Fb, st, sf):
    Cout = [8, 64, 256][(Fb + st + sf) % 3]
    _c1_case(parity, 2, 7, Fb, Cout, st, sf, seed=Fb * 10 + st + sf)


@pytest.mark.parametrize("T", [1, 2, 9])
@pytest.mark.parametrize("Cout", [8, 64, 256])
def test_conv3x3_c1_short_inputs(parity, T, Cout):
    _c1_case(parity, 3, T, 83, Cout, 2, 2, seed=T + Cout)


def test_conv3x3_c1_35s_layer(parity):
    """One 35 s utterance of 80-bin fbank frames (3500 frames) through the conv front's first layer."""
    _c1_case(parity, 1, 3500, 80, 64, 2, 2, seed=31)


# -------------------------------------------------------------------------------------------------------------- optimizer
@pytest.mark.parametrize("n", [1, 3, 4, 5, 100003, 30000000])
def test_sumsq(parity, n):
    g = torch.randn(n, generator=_gen(n % 1000), device="cuda") * 3
    ob, out = _boxed((1,), F32, init=torch.full((1,), 7.0, device="cuda"))
    assert _L().esp_sumsq_f32(_p(g), n, _p(out), _stream()) == 0
    r = K.sumsq(g)
    torch.cuda.synchronize()
    _untouched(ob, out, "sumsq")
    _check(parity, "sumsq n=%d" % n, out[0], r.out, r.out_mag, TAU_SUMSQ)


def _adam_run(parity, tag, n, steps, lr, b1, b2, wd, clip, denom, denom_dev=False, hyper=False, gscale=1.0, clips=None):
    L = _L()
    gen = _gen(n)
    p32 = torch.randn(n, generator=gen, device="cuda")
    m = torch.randn(n, generator=gen, device="cuda") * 1e-2
    v = torch.rand(n, generator=gen, device="cuda") * 1e-4
    p16b, p16 = _boxed((n,), BF)
    gnb, gn = _boxed((1,), F32)
    ss = torch.zeros(1, device="cuda")
    dd = torch.tensor([denom], device="cuda", dtype=F32) if denom_dev else None
    for step in steps:
        g = torch.randn(n, generator=gen, device="cuda") * gscale
        assert L.esp_sumsq_f32(_p(g), n, _p(ss), _stream()) == 0
        hy = torch.tensor([lr, float(step)], device="cuda", dtype=F32) if hyper else None
        p0, m0, v0 = p32.clone(), m.clone(), v.clone()
        assert L.esp_adam_step(_p(p32), _p(m), _p(v), _p(g), _p(p16), n, 0.0 if hyper else lr, b1, b2, 1e-8, wd,
                               0 if hyper else step, _p(ss), _p(dd), 0.0 if denom_dev else denom, clip, _p(gn), _p(hy),
                               _stream()) == 0
        r = K.adam_step(p0, m0, v0, g, float(np.float32(lr)), b1, b2, 1e-8, wd, step, float(ss), denom, clip)
        torch.cuda.synchronize()
        _untouched(p16b, p16, tag + " p16")
        _untouched(gnb, gn, tag + " gnorm")
        t = "%s step %d" % (tag, step)
        _check(parity, t + " p", p32, r.p, r.p_mag, TAU_ADAM, r.p_fl)
        _check(parity, t + " m", m, r.m, r.m_mag, TAU_ADAM)
        _check(parity, t + " v", v, r.v, r.v_mag, TAU_ADAM)
        _check(parity, t + " gnorm", gn[0], torch.tensor(r.gnorm, dtype=F64, device="cuda"), abs(r.gnorm), TAU_ADAM)
        assert torch.equal(p16.view(torch.int16), p32.to(BF).view(torch.int16)), t + ": p16 != RN(p32)"
        if clips is not None:
            assert (r.coef < 1) == clips, t + ": clipping should be %s" % ("active" if clips else "inactive")


@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("clip_active", [False, True])
def test_adam_steps_with_clipping(parity, clip_active, wd):
    """Six steps; the gradient norm sits far above (clipping active) or below (inactive) clip_norm = 25."""
    n = 4099
    _adam_run(parity, "adam clip=%d wd=%g" % (clip_active, wd), n, range(1, 7), 5e-4, 0.9, 0.98, wd, 25.0, 8.0,
              gscale=10.0 if clip_active else 0.01, clips=clip_active)


@pytest.mark.parametrize("denom", [0.0, 3.0])
@pytest.mark.parametrize("denom_dev", [False, True])
def test_adam_denominator(parity, denom_dev, denom):
    _adam_run(parity, "adam denom=%g dev=%d" % (denom, denom_dev), 1027, range(1, 4), 1e-3, 0.9, 0.98, 0.01, 1.0, denom,
              denom_dev=denom_dev, gscale=1.0)


def test_adam_hyper_dev(parity):
    _adam_run(parity, "adam hyper_dev", 1027, [1, 2, 3, 250, 251], 7e-4, 0.9, 0.98, 0.0, 0.0, 5.0, hyper=True)


@pytest.mark.parametrize("b2", [0.98, 0.999])
@pytest.mark.parametrize("step", [1, 1000, 100000])
def test_adam_bias_correction(parity, step, b2):
    _adam_run(parity, "adam step=%d b2=%g" % (step, b2), 2053, [step], 1e-3, 0.9, b2, 0.0, 0.0, 1.0)


def test_casts_bit_exact(parity):
    """f32 -> bf16 and bf16 -> f32 against torch's own device casts, bit for bit: NaNs (with payloads and sign), +-inf,
    -0, fp32 and bf16 subnormals, exact ties (even and odd), values that overflow to inf, and every bf16 pattern."""
    ints = [0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FBFFFFF, 0xFFFFFFFF, 0x7F800000, 0xFF800000, 0x80000000, 0x00000000,
            0x00000001, 0x807FFFFF, 0x00400000, 0x00008000, 0x00018000, 0x3F808000, 0x3F818000, 0xBF808000, 0x3F80C000,
            0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000, 0x7F7F7FFF, 0x00800000, 0x0000FFFF]
    special = torch.tensor(np.array(ints, dtype=np.uint32).view(np.int32), device="cuda").view(F32)
    rnd = torch.randint(-2 ** 31, 2 ** 31 - 1, (1 << 20,), generator=_gen(41), device="cuda", dtype=torch.int64)
    x = torch.cat([special, rnd.to(torch.int32).view(F32)])
    n = x.numel()
    yb, y = _boxed((n,), BF)
    assert _L().esp_cast_f32_bf16(_p(x), n, _p(y), _stream()) == 0
    allbf = torch.arange(-32768, 32768, device="cuda", dtype=torch.int32).to(torch.int16).view(BF)
    fb, f = _boxed((65536,), F32)
    assert _L().esp_cast_bf16_f32(_p(allbf), 65536, _p(f), _stream()) == 0
    torch.cuda.synchronize()
    _untouched(yb, y, "cast f32->bf16")
    _untouched(fb, f, "cast bf16->f32")
    assert torch.equal(y.view(torch.int16), x.to(BF).view(torch.int16))
    assert torch.equal(f.view(torch.int32), allbf.float().view(torch.int32))
    parity("casts bit-exact", 0.0, 0.0)


# --------------------------------------------------------------------------------- compositions at the bench shapes
def _ragged(B, T):
    return torch.tensor([T - (b * 37) % (T // 2) for b in range(B)], dtype=torch.int32, device="cuda")


def test_conv_module_chain_against_autograd(parity):
    """glu_dwconv -> bn_finalize -> bn_silu and back, d = 512, k = 31, B = 24, T' = 275, padded frames zeroed (ragged):
    every output and gradient against float64 autograd of F.glu, grouped conv1d, batch-statistics BatchNorm and SiLU."""
    ops = _ops()
    B, T, C_, k = 24, 275, 512, 31
    lens = _ragged(B, T)
    valid = (torch.arange(T, device="cuda")[None, :] < lens[:, None].long())[:, :, None]
    g = (_glu_input(B, T, C_, 51) * valid).contiguous()
    w = _rand((C_, k), 52, 0.2)
    gm, bt = _rand(C_, 53, 0.5, 1.0), _rand(C_, 54, 0.3)
    dz = _rand((B, T, C_), 55)
    y, st = ops.glu_dwconv_fwd(g, w)
    rm, rv = torch.zeros(C_, device="cuda"), torch.ones(C_, device="cuda")
    mr = ops.bn_finalize(st, B * T, C_, 1e-5, 0.1, rm, rv, True)
    z = ops.bn_act_fwd(y, mr, gm, bt, 1)
    dg_, db_ = torch.zeros(C_, device="cuda"), torch.zeros(C_, device="cuda")
    dy = ops.bn_act_bwd(dz, y, mr, gm, bt, dg_, db_, 1)
    dw = torch.zeros(C_, k, device="cuda")
    dgl = ops.glu_dwconv_bwd(dy, g, w, dw)
    g64 = g.to(F64).requires_grad_(True)
    w64, gm64, bt64 = (t.to(F64).requires_grad_(True) for t in (w, gm, bt))
    rm64, rv64 = torch.zeros(C_, device="cuda", dtype=F64), torch.ones(C_, device="cuda", dtype=F64)
    c = F.conv1d(F.glu(g64, -1).transpose(1, 2), w64[:, None, :], padding=k // 2, groups=C_)
    z64 = F.silu(F.batch_norm(c, rm64, rv64, gm64, bt64, training=True, momentum=0.1, eps=1e-5)).transpose(1, 2)
    z64.backward(dz.to(F64))
    _rel(parity, "conv module z", z, z64.detach())
    _rel(parity, "conv module running mean", rm, rm64)
    _rel(parity, "conv module running var", rv, rv64)
    _rel(parity, "conv module dg", dgl, g64.grad)
    _rel(parity, "conv module dw", dw, w64.grad)
    _rel(parity, "conv module dgamma", dg_, gm64.grad)
    _rel(parity, "conv module dbeta", db_, bt64.grad)


def test_conv_front_layer1_against_autograd(parity):
    """conv3x3_c1 (stride 2) -> BatchNorm with the conv bias as pre_bias -> ReLU and back, at B = 24, T = 1100, F = 80,
    C = 64: every output and gradient against float64 autograd of F.conv2d (with bias), batch_norm and relu."""
    ops = _ops()
    B, T, Fb, C_ = 24, 1100, 80, 64
    x = _rand((B, T, Fb), 61, 1.5)
    w, bias = _rand((C_, 3, 3), 62, 0.4), _rand(C_, 63, 0.3)
    gm, bt = _rand(C_, 64, 0.5, 1.0), _rand(C_, 65, 0.3)
    y = ops.conv3x3_fwd(x, w, (2, 2))
    st = ops.bn_stats(y, C_, bias)
    R = y.numel() // C_
    mr = ops.bn_finalize(st, R, C_, 1e-5, 0.1, None, None, True)
    z = ops.bn_act_fwd(y, mr, gm, bt, 2, bias)
    dz = _rand(z.shape, 66)
    dg_, db_ = torch.zeros(C_, device="cuda"), torch.zeros(C_, device="cuda")
    dy = ops.bn_act_bwd(dz, y, mr, gm, bt, dg_, db_, 2, bias)
    dw = torch.zeros(C_, 3, 3, device="cuda")
    ops.conv3x3_wgrad(dy, x, dw, (2, 2))
    x64 = x.to(F64)[:, None]
    ybf = (y.float() + bias.float()).to(BF).to(F64).permute(0, 3, 1, 2)  # what the BatchNorm normalises

    def reference(rounded):
        w64, b64, gm64, bt64 = (t.to(F64).requires_grad_(True) for t in (w, bias, gm, bt))
        c = F.conv2d(x64, w64[:, None], b64, (2, 2), 1)
        if rounded:  # the same conv and its gradient, with the value of the documented bf16(y + bias)
            c = c + (ybf - c).detach()
        z64 = torch.relu(F.batch_norm(c, None, None, gm64, bt64, training=True, eps=1e-5)).permute(0, 2, 3, 1)
        z64.backward(dz.to(F64))
        return z64.detach(), w64.grad, b64.grad, gm64.grad, bt64.grad
    z64, dw64, db64, dgm64, dbt64 = reference(False)
    _rel(parity, "conv front z", z, z64)
    parity("conv front dbias / |dw| (identically 0 through batch statistics)", float(db64.norm() / dw64.norm()), 1e-9)
    # dw, dgamma and dbeta are cancelling sums (the batch-statistics backward leaves dy nearly orthogonal to y): their distance
    # from the float64 gradients is set by the bf16 rounding of y + bias.  Against autograd through that same rounding
    # they are at the level of every other gradient.
    _rel(parity, "conv front dw", dw, dw64, GRAD_REL_FRONT)
    _rel(parity, "conv front dgamma", dg_, dgm64, GRAD_REL_FRONT)
    _rel(parity, "conv front dbeta", db_, dbt64, GRAD_REL_FRONT)
    _, dwr, _, dgmr, dbtr = reference(True)
    _rel(parity, "conv front dw (through bf16(y + bias))", dw, dwr)
    _rel(parity, "conv front dgamma (through bf16(y + bias))", dg_, dgmr)
    _rel(parity, "conv front dbeta (through bf16(y + bias))", db_, dbtr)


def test_layer_norm_against_autograd(parity):
    ops = _ops()
    B, T, d = 24, 275, 512
    R = B * T
    lens = _ragged(B, T)
    x, gm, bt = _rand((R, d), 71), _rand(d, 72, 0.5, 1.0), _rand(d, 73, 0.3)
    dy = _rand((R, d), 74)
    y, mean, rstd = ops.layer_norm_fwd(x, gm, bt, 1e-5, lens, T)
    dg_, db_ = torch.zeros(d, device="cuda"), torch.zeros(d, device="cuda")
    dx = ops.layer_norm_bwd(dy, x, mean, rstd, gm, dg_, db_, lens=lens, T=T)
    valid = (torch.arange(R, device="cuda") % T < lens.long()[torch.arange(R, device="cuda") // T])[:, None]
    x64, gm64, bt64 = (t.to(F64).requires_grad_(True) for t in (x, gm, bt))
    y64 = F.layer_norm(x64, (d,), gm64, bt64, 1e-5) * valid
    y64.backward(dy.to(F64))
    _rel(parity, "layer norm y", y, y64.detach())
    _rel(parity, "layer norm dx", dx, x64.grad)
    _rel(parity, "layer norm dgamma", dg_, gm64.grad)
    _rel(parity, "layer norm dbeta", db_, bt64.grad)


# ------------------------------------------------------------------------------------------------------ host refusals
def _refused(call, what, match):
    lib = _lib()
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    assert call() != 0, what + " was accepted"
    assert match in _L().esp_last_error().decode(), _L().esp_last_error().decode()
    assert lib.launch_count() == n0, what + ": launched a kernel"


def test_host_refusals(parity):
    L, s = _L(), _stream()
    g = _rand((1, 16, 2 * 144), 81)
    w144 = _rand((144, 3), 82)
    yb, y = _boxed((1, 16, 144))
    st = torch.zeros(2, 144, device="cuda", dtype=F64)
    _refused(lambda: L.esp_glu_dwconv_fwd(_p(g), _p(w144), 1, 16, 144, 3, _p(y), _p(st), s), "dwconv C=144", "multiple of 64")
    _refused(lambda: L.esp_glu_dwconv_bwd(_p(y), _p(g), _p(w144), 1, 16, 144, 3, _p(g), _p(st), s), "dwconv bwd C=144",
             "unsupported depthwise")
    g64 = _rand((1, 16, 128), 83)
    w64 = _rand((64, 33), 84)
    for kk in (4, 33):
        _refused(lambda: L.esp_glu_dwconv_fwd(_p(g64), _p(w64), 1, 16, 64, kk, _p(y), _p(st), s), "dwconv k=%d" % kk,
                 "odd and <= 31")
        _refused(lambda: L.esp_glu_dwconv_bwd(_p(y), _p(g64), _p(w64), 1, 16, 64, kk, _p(g), _p(st), s),
                 "dwconv bwd k=%d" % kk, "unsupported depthwise")
    x = _rand((12, 2056), 85)
    gm = _rand(2056, 86)
    mb, mean = _boxed((12,), F32)
    for dd in (12, 2056):
        _refused(lambda: L.esp_layer_norm_fwd(_p(x), _p(gm), _p(gm), 1e-5, 12, dd, _p(y), _p(mean), _p(mean), None, 0, 0.0, 0,
                                              None, s), "LayerNorm d=%d" % dd, "unsupported")
        _refused(lambda: L.esp_layer_norm_bwd2(_p(x), _p(x), _p(mean), _p(mean), _p(gm), None, 12, dd, _p(y), _p(mean), _p(mean),
                                               None, 0, 0.0, 0, None, None, 0.0, 0, 1.0, s), "LayerNorm bwd d=%d" % dd,
                 "unsupported")
    # lens needs rows [B, T]: T = 0 (the wrappers' default) and T not dividing R are refused before any launch
    lens = torch.tensor([3, 2, 4], dtype=torch.int32, device="cuda")
    for T in (0, 5):
        _refused(lambda: L.esp_layer_norm_fwd(_p(x), _p(gm), _p(gm), 1e-5, 12, 64, _p(y), _p(mean), _p(mean), _p(lens), T, 0.0,
                                              0, None, s), "LayerNorm lens T=%d" % T, "T >= 1 dividing R")
        _refused(lambda: L.esp_layer_norm_bwd2(_p(x), _p(x), _p(mean), _p(mean), _p(gm), None, 12, 64, _p(y), _p(mean),
                                               _p(mean), _p(lens), T, 0.0, 0, None, None, 0.0, 0, 1.0, s),
                 "LayerNorm bwd lens T=%d" % T, "T >= 1 dividing R")
    xb = _rand((10, 24), 87)
    _refused(lambda: L.esp_bn_stats(_p(xb), None, 10, 24, _p(st), s), "bn_stats C=24", "C/8 must divide 256")
    mr = torch.zeros(2, 64, device="cuda")
    x64 = _rand((10, 64), 88)
    _refused(lambda: L.esp_bn_act_fwd(_p(x64), None, 10, 64, _p(mr), _p(gm), _p(gm), 0, _p(x64), s), "bn_act act=0",
             "act must be 1")
    ws = torch.zeros(3, 64, device="cuda", dtype=F64)
    _refused(lambda: L.esp_bn_act_bwd(_p(x64), _p(x64), None, 10, 64, _p(mr), _p(gm), _p(gm), 0, _p(ws), _p(x64), _p(mr),
                                      _p(mr), s), "bn_act_bwd act=0", "act must be 1")
    # bn_finalize in training over zero rows would write 0/0 into the running statistics
    rmb, rm = _boxed((64,), F32, init=torch.zeros(64, device="cuda"))
    rvb, rv = _boxed((64,), F32, init=torch.ones(64, device="cuda"))
    mrb, mr2 = _boxed((2, 64), F32)
    st64 = torch.zeros(2, 64, device="cuda", dtype=F64)
    _refused(lambda: L.esp_bn_finalize(_p(st64), 0, 64, 1e-5, 0.1, _p(rm), _p(rv), 1, _p(mr2), s), "bn_finalize R=0",
             "0 rows")
    # the first conv's weight gradient with a time stride of 0
    xc = _rand((1, 8, 8), 89)
    dwb, dw = _boxed((8, 3, 3), F32, init=torch.zeros(8, 3, 3, device="cuda"))
    _refused(lambda: L.esp_conv3x3_c1_wgrad(_p(xc), _p(xc), _p(dw), 1, 8, 8, 8, 0, 1, s), "conv3x3_c1 wgrad st=0",
             "stride")
    torch.cuda.synchronize()
    _untouched(yb, y[:0], "refused y")
    _untouched(mb, mean[:0], "refused mean")
    _untouched(mrb, mr2[:0], "refused mr")
    assert torch.equal(rm, torch.zeros(64, device="cuda")) and torch.equal(rv, torch.ones(64, device="cuda"))
    assert torch.equal(dw, torch.zeros(8, 3, 3, device="cuda"))
    _untouched(rmb, rm, "refused run_mean")
    _untouched(dwb, dw, "refused dw")
    parity("host refusals", 0.0, 0.0)
