"""Float64 statements of the block kernels of csrc/elementwise.cu and csrc/optim.cu: LayerNorm (with the fused dx2 output),
column sums, q preparation, row masking, GLU + depthwise conv (+ BatchNorm statistics), BatchNorm + SiLU / ReLU, the
one-input-channel first convolution, and the optimizer (squared norm, fused clip + Adam, casts).

TEST INFRASTRUCTURE ONLY.  Each function has the signature of its espresso_b200.ops wrapper and works from the kernel's
own bf16 inputs, widened exactly; dropout masks come from oracle/dropout_rng.py, so they are the kernels' masks bit for
bit.  Nothing is written: every function returns float64 results.

Rounding points.  The statements model the roundings the kernels document, and no others:
  * the GLU output is bf16 before the depthwise conv, and the conv output is bf16 before its statistics;
  * the pre_bias sum bf16(x + b) and the BatchNorm output bf16(bn) before the activation;
  * q preparation rounds bf16(q + u) before scaling;
  * dx2 = dropout(bf16(dx)) * scale2.
A value rounded to bf16 inside a kernel is stated as RN(x64).  The kernel rounds its own fp32 value, which lies within
some delta of x64, so the two roundings can differ by one bf16 ulp where x64 lies within delta of a rounding midpoint.
`Rounded` carries that possible difference, `flip = RN(x64 + delta) - RN(x64 - delta)`, and every later step propagates
it into its bound.  Elsewhere the rounded value is exact, so a dropped or an added rounding point moves outputs by
2^-9 of their size, far outside any fp32-level bound.

Bounds.  Every result carries the magnitude its bound is built from, as in oracle/gemm64.py and oracle/attn64.py:
  fp32 outputs   |x - x64| <= tau * mag + fl
  bf16 outputs   |x - x64| <= 2^-8 |x64| + (1 + 2^-8) (tau * mag + fl)
fl collects the terms that are not fp32 reduction error: the propagated rounding flips and, where a sigmoid is
involved, apx * SIG_ABS.  `sigmoidf_` is __fdividef(1, 1 + __expf(-x)): with __expf's relative error of
(2 + 1.173 |x|) 2^-23 and __fdividef's 2 ulp, |sigmoid~(x) - sigmoid(x)| <= sigmoid (1 - sigmoid) (2 + 1.173 |x|) 2^-23
+ 3 * 2^-23 sigmoid < 2^-21 = SIG_ABS for every x (at most 0.6 * 2^-23 from the first term), and apx is the
coefficient of that error in each output.
The Adam statement is fairseq's Adam.step with the bias corrections in Python doubles; the kernel forms them in fp32
with powf from the fp32 betas, and `pow_err` states how far that moves the step size.
"""
import math

import numpy as np
import torch

from oracle import dropout_rng as _rng
from oracle import gemm64 as _g64

F64, F32, BF = torch.float64, torch.float32, torch.bfloat16
U32 = 2.0 ** -24            # fp32 unit roundoff
BF_REL = 2.0 ** -8          # half a bf16 ulp, relative
SIG_ABS = 2.0 ** -21        # |sigmoid~ - sigmoid| of sigmoidf_ (see the module docstring)
SILU_LIP = 1.1              # |silu'| <= 1.0998


class Result:
    """Fields by name; each value x comes with x_mag (tau scale) and x_fl (absolute terms), see the module docstring."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def rn(x):
    """Round-to-nearest-even to bf16 of a float64 tensor, directly (no fp32 step), as float64: 8 significant bits, and the
    subnormal spacing 2^-133 below 2^-126."""
    _, e = torch.frexp(x)
    ulp = torch.ldexp(torch.ones_like(x), e.clamp_min(-125) - 8)
    return torch.round(x / ulp) * ulp


def rounded(x, delta):
    """RN(x) and the largest difference from it of RN(y) for |y - x| <= delta."""
    r = rn(x)
    return r, torch.maximum((rn(x + delta) - r).abs(), (r - rn(x - delta)).abs())


def tau_reached(got, val, mag, fl=0.0, bf16=False):
    """Smallest tau with every element of got inside the bound (0 when the flip / sigmoid terms cover all of them).
    An element with zero magnitude must sit inside its non-tau terms."""
    val = val.to(F64)
    err = (got.to(F64) - val).abs()
    if not torch.is_tensor(fl):
        fl = torch.full_like(val, float(fl))
    if bf16:
        err = (err - BF_REL * val.abs()) / (1 + BF_REL)
    ex = err - fl
    mag = mag.to(F64).expand_as(ex) if torch.is_tensor(mag) else torch.full_like(ex, float(mag))
    zero = mag == 0
    if bool((ex[zero] > 0).any()):
        return float("inf")
    if ex.numel() == 0:
        return 0.0
    return float((ex.clamp_min(0) / torch.where(zero, torch.ones_like(mag), mag)).max())


def dscale(p, scale=1.0):
    """The kernels' fp32 rescale of kept elements: fp32(fp32(scale * 65536) / (65536 - thresh)), `scale` at p = 0."""
    if _rng.thresh(p) == 0:
        return float(np.float32(scale))
    return float(np.float32(np.float32(np.float32(scale) * np.float32(65536.0)) / np.float32(65536.0 - _rng.thresh(p))))


def keep(seed, R, N, p, device, device_seed=0):
    """Keep mask of the row-major [R, N] block (index r * N + c); all True at thresh(p) == 0."""
    if _rng.thresh(p) == 0:
        return torch.ones(R, N, dtype=torch.bool, device=device)
    return _rng.keep_mask(_rng.combine_seed(seed, device_seed), _rng.row_major_index(R, N), p).to(device)


def _row_valid(R, lens, T, device):
    if lens is None:
        return torch.ones(R, dtype=torch.bool, device=device)
    r = torch.arange(R, device=device)
    return (r % T) < lens.to(device).long()[r // T]


# ------------------------------------------------------------------------------------------------------------ LayerNorm
def layer_norm_fwd(x, gamma, beta, eps=1e-5, lens=None, T=0, drop_p=0.0, seed=0, device_seed=0):
    """y = dropout(LN(x)) on rows t < lens[b], 0 on the others; mean, rstd per row.
    mag: |x - mean| + mean|x| (the fp32 mean's error reaches every element) times rstd |gamma|, + |beta|, through the
    dropout scale.  mean_mag = mean|x|, rstd_mag = rstd (relative)."""
    xd, gd, bd = x.to(F64), gamma.to(F64), beta.to(F64)
    R, d = xd.shape
    mean = xd.mean(-1)
    c = xd - mean[:, None]
    var = (c * c).mean(-1)
    rstd = 1.0 / torch.sqrt(var + eps)
    y = c * rstd[:, None] * gd + bd
    amean = xd.abs().mean(-1)
    mag = (c.abs() + amean[:, None]) * rstd[:, None] * gd.abs() + bd.abs()
    k = keep(seed, R, d, drop_p, x.device, device_seed)
    s = dscale(drop_p)
    y = torch.where(k, y * s, torch.zeros_like(y))
    mag = torch.where(k, mag * s, torch.zeros_like(mag))
    valid = _row_valid(R, lens, T, x.device)[:, None]
    y, mag = y * valid, mag * valid
    return Result(y=y, y_mag=mag, mean=mean, mean_mag=amean, rstd=rstd, rstd_mag=rstd)


def layer_norm_bwd(dy, x, mean, rstd, gamma, dgamma_acc, dbeta_acc, dres=None, lens=None, T=0, drop_p=0.0, seed=0,
                   next_drop=None, device_seed=0):
    """From the kernel's own fp32 mean / rstd:  dyv = dropout(dy) on valid rows, h = (x - mean) rstd,
    dx = rstd (g dyv - mean(g dyv) - h mean(g dyv h)) + dres;  dgamma = dgamma0 + sum dyv h;  dbeta = dbeta0 + sum dyv.
    next_drop = (p2, seed2, scale2) states dx2 from the kernel's own dx: `dx2_of(dx_got)` (bit-exact form)."""
    xd, gd = x.to(F64), gamma.to(F64)
    R, d = xd.shape
    m, rs = mean.to(F64)[:, None], rstd.to(F64)[:, None]
    k = keep(seed, R, d, drop_p, x.device, device_seed)
    dyv = torch.where(k, dy.to(F64) * dscale(drop_p), torch.zeros(R, d, dtype=F64, device=x.device))
    dyv = dyv * _row_valid(R, lens, T, x.device)[:, None]
    h = (xd - m) * rs
    g = dyv * gd
    s1, s2 = g.mean(-1, keepdim=True), (g * h).mean(-1, keepdim=True)
    dx = rs * (g - s1 - h * s2)
    mag = rs * (g.abs() + g.abs().mean(-1, keepdim=True) + h.abs() * (g * h).abs().mean(-1, keepdim=True))
    if dres is not None:
        dx, mag = dx + dres.to(F64), mag + dres.to(F64).abs()
    dg0, db0 = dgamma_acc.to(F64), dbeta_acc.to(F64)
    out = Result(dx=dx, dx_mag=mag, dgamma=dg0 + (dyv * h).sum(0), dgamma_mag=dg0.abs() + (dyv * h).abs().sum(0),
                 dbeta=db0 + dyv.sum(0), dbeta_mag=db0.abs() + dyv.abs().sum(0))
    if next_drop is not None:
        p2, seed2, scale2 = next_drop
        k2 = keep(seed2, R, d, p2, x.device, device_seed)
        s = dscale(p2, scale2)

        def dx2_of(dx_got):
            v = (dx_got.to(F32) * torch.tensor(s, dtype=F32, device=dx_got.device)).to(BF)
            return torch.where(k2, v, torch.zeros_like(v))
        out.dx2_of = dx2_of
    return out


# ------------------------------------------------------------------------------------------------- column sums, q prep
def colsum(x, out_acc, scale=1.0):
    """out = out0 + scale * sum_r x[r, :]."""
    xd, o = x.to(F64), out_acc.to(F64)
    return Result(out=o + scale * xd.sum(0), out_mag=o.abs() + abs(scale) * xd.abs().sum(0))


def _f32(x):
    return x.to(F32).to(F64)


def qprep_fwd(q, u, v, scale):
    """q_u = bf16(fp32(bf16(fp32(q + u)) * s)), q_v likewise: every step is one exactly stated rounding."""
    s = float(np.float32(scale))
    qd = q.to(F64)
    qu = rn(_f32(rn(_f32(qd + u.to(F64))) * s))
    qv = rn(_f32(rn(_f32(qd + v.to(F64))) * s))
    return qu.to(BF), qv.to(BF)


def qprep_bwd(dqu, dqv, scale):
    """dq = bf16(fp32(s * fp32(dqu + dqv)))."""
    return rn(_f32(float(np.float32(scale)) * _f32(dqu.to(F64) + dqv.to(F64)))).to(BF)


def mask_rows(x, lens):
    B, T, _ = x.shape
    keep_t = torch.arange(T, device=x.device)[None, :] < lens.to(x.device).long()[:, None]
    return torch.where(keep_t[:, :, None], x, torch.zeros_like(x))


# ------------------------------------------------------------------------------------------------ GLU + depthwise conv
def _sig(x):
    return torch.sigmoid(x)


def glu(g):
    """RN(a sigmoid(gate)) with its flip: the kernel's fp32 a * sigmoid~(gate) is within |a| SIG_ABS + 2^-23 |glu|."""
    C = g.shape[-1] // 2
    a, gate = g[..., :C].to(F64), g[..., C:].to(F64)
    v = a * _sig(gate)
    return rounded(v, a.abs() * SIG_ABS + 2 * U32 * v.abs())


def _dwconv(x, w):
    """Depthwise correlation along T with 'same' zero padding: y[b, t, c] = sum_k w[c, k] x[b, t + k - k//2, c]."""
    B, T, C = x.shape
    k = w.shape[1]
    h = k // 2
    xp = torch.nn.functional.pad(x, (0, 0, h, h))
    y = torch.zeros(B, T, C, dtype=F64, device=x.device)
    for j in range(k):
        y += xp[:, j:j + T, :] * w[:, j]
    return y


def glu_dwconv_fwd(g, w):
    """y = RN(dwconv(RN(GLU(g)))).  y_mag / y_fl bound the unrounded conv (the bf16 output rule adds the rounding);
    y_fl carries the GLU flips through |w|.  stats_of(y_got): the per-channel sum and sum of squares of the kernel's own
    bf16 output over all B*T rows (value, magnitude)."""
    wd = w.to(F64)
    gl, gfl = glu(g)
    y = _dwconv(gl, wd)
    mag = _dwconv(gl.abs(), wd.abs())
    fl = _dwconv(gfl, wd.abs())

    def stats_of(y_got):
        yv = y_got.to(F64).reshape(-1, y_got.shape[-1])
        st = torch.stack([yv.sum(0), (yv * yv).sum(0)])
        return st, torch.stack([yv.abs().sum(0), (yv * yv).sum(0)])
    return Result(y=y, y_mag=mag, y_fl=fl, glu=gl, stats_of=stats_of)


def glu_dwconv_bwd(dy, g, w, dw_acc):
    """dglu[t] = sum_k w[k] dy[t - k + k//2] (fp32, not rounded);  dg_a = dglu sigmoid(gate),
    dg_gate = dglu a sigmoid (1 - sigmoid);  dw = dw0 + sum_{b,t} dy[t] RN(glu)[t + k - k//2]."""
    C = g.shape[-1] // 2
    a, gate = g[..., :C].to(F64), g[..., C:].to(F64)
    wd, dyd = w.to(F64), dy.to(F64)
    wf = wd.flip(1)
    dglu = _dwconv(dyd, wf)
    dmag = _dwconv(dyd.abs(), wf.abs())
    s = _sig(gate)
    sp = s * (1 - s)
    da = dglu * s
    dgt = dglu * a * sp
    gl, gfl = glu(g)
    B, T, _ = dy.shape
    k = w.shape[1]
    h = k // 2
    glp = torch.nn.functional.pad(gl, (0, 0, h, h))
    flp = torch.nn.functional.pad(gfl, (0, 0, h, h))
    dw0 = dw_acc.to(F64)
    dw, dwm, dwf = dw0.clone(), dw0.abs(), torch.zeros_like(dw0)
    for j in range(k):
        dw[:, j] += (dyd * glp[:, j:j + T, :]).sum((0, 1))
        dwm[:, j] += (dyd.abs() * glp[:, j:j + T, :].abs()).sum((0, 1))
        dwf[:, j] += (dyd.abs() * flp[:, j:j + T, :]).sum((0, 1))
    dg = torch.cat([da, dgt], -1)
    dg_mag = torch.cat([dmag * s, dmag * a.abs() * sp], -1)
    dg_fl = torch.cat([dglu.abs() * SIG_ABS, (dglu * a).abs() * SIG_ABS], -1)  # |d(s(1-s))/ds| = |1 - 2s| <= 1
    return Result(dg=dg, dg_mag=dg_mag, dg_fl=dg_fl, dw=dw, dw_mag=dwm, dw_fl=dwf)


# ---------------------------------------------------------------------------------------------------------- BatchNorm
def pre(y, pre_bias):
    """The normalised tensor: y, or RN(y + pre_bias[c]) with its flip (the fp32 sum is within 2^-23 of the exact one)."""
    yd = y.to(F64)
    if pre_bias is None:
        return yd, torch.zeros_like(yd)
    v = yd + pre_bias.to(F64)
    return rounded(v, 2 * U32 * v.abs())


def bn_stats(x, C_, pre_bias=None):
    """stats [2, C] = per-channel sum and sum of squares of pre(x); magnitudes; fl of the pre_bias flips."""
    v, fl = pre(x, pre_bias)
    v, fl = v.reshape(-1, C_), fl.reshape(-1, C_)
    st = torch.stack([v.sum(0), (v * v).sum(0)])
    mag = torch.stack([v.abs().sum(0), (v * v).sum(0)])
    stfl = torch.stack([fl.sum(0), (fl * (2 * v.abs() + fl)).sum(0)])
    return Result(stats=st, stats_mag=mag, stats_fl=stfl)


def bn_finalize(stats, R, C_, eps, momentum, run_mean, run_var, training):
    """Training: mean = s1 / R, var = max(s2 / R - mean^2, 0), rstd = 1 / sqrt(var + eps); running mean and variance
    (1 - momentum) r + momentum * (mean, var R / (R - 1)) (var itself at R = 1).  Eval: the running statistics.
    Magnitudes: mean (one fp32 rounding), rstd (relative), running terms |(1 - m) r| + |m x|."""
    if training:
        s = stats.to(F64)
        mean = s[0] / R
        var = (s[1] / R - mean * mean).clamp_min(0)
        rstd = 1.0 / torch.sqrt(var + eps)
        out = Result(mean=mean, mean_mag=mean.abs(), rstd=rstd, rstd_mag=rstd)
        if run_mean is not None:
            unb = var * R / (R - 1) if R > 1 else var
            rm, rv = run_mean.to(F64), run_var.to(F64)
            out.run_mean = (1 - momentum) * rm + momentum * mean
            out.run_mean_mag = (1 - momentum) * rm.abs() + momentum * mean.abs()
            out.run_var = (1 - momentum) * rv + momentum * unb
            out.run_var_mag = (1 - momentum) * rv.abs() + momentum * unb
        return out
    rv = run_var.to(F64)
    rstd = 1.0 / torch.sqrt(rv + eps)
    return Result(mean=run_mean.to(F64), mean_mag=torch.zeros_like(rv), rstd=rstd, rstd_mag=rstd)


BN_ACT_SILU, BN_ACT_RELU = 1, 2


def _bn(y, mr, gamma, beta, pre_bias):
    """xh = (v - mean) rstd from the kernel's fp32 mean / rstd, bn = RN(xh gamma + beta) with its flip (the fp32 form is
    within 4 * 2^-24 (|xh gamma| + |beta|) + |rstd gamma| * the pre_bias flip)."""
    C = y.shape[-1]
    v, vfl = pre(y, pre_bias)
    v, vfl = v.reshape(-1, C), vfl.reshape(-1, C)
    mu, rs = mr[0].to(F64), mr[1].to(F64)
    gd, bd = gamma.to(F64), beta.to(F64)
    xh = (v - mu) * rs
    pre_bn = xh * gd + bd
    delta = 4 * U32 * ((xh * gd).abs() + bd.abs()) + (rs * gd).abs() * vfl
    bn, bfl = rounded(pre_bn, delta)
    return xh, bn, bfl, (rs * vfl)


def _act(x, act):
    return x * _sig(x) if act == BN_ACT_SILU else x.clamp_min(0)


def _act_grad(x, act):
    if act == BN_ACT_SILU:
        s = _sig(x)
        return s * (1 + x * (1 - s))
    return (x > 0).to(F64)  # strict: bn == 0 passes no gradient


def bn_act_fwd(y, mr, gamma, beta, act=BN_ACT_SILU, pre_bias=None):
    """z = act(RN(bn)) (bf16 output rule on z).  z_fl: the bn flip through act (|act'| <= 1.1) and, for SiLU,
    |bn| SIG_ABS; z_mag = |z| (the fp32 product of SiLU; ReLU is exact given bn)."""
    _, bn, bfl, _ = _bn(y, mr, gamma, beta, pre_bias)
    z = _act(bn, act)
    fl = SILU_LIP * bfl + (bn.abs() * SIG_ABS if act == BN_ACT_SILU else 0)
    return Result(z=z.reshape(y.shape), z_mag=z.abs().reshape(y.shape), z_fl=fl.reshape(y.shape), bn=bn)


def bn_act_bwd(dz, y, mr, gamma, beta, dgamma_acc, dbeta_acc, act=BN_ACT_SILU, pre_bias=None):
    """dbn = dz act'(RN(bn)); s1 = sum dbn, s2 = sum dbn xh over all R rows; dy = gamma rstd (dbn - s1/R - xh s2/R);
    dgamma = dgamma0 + s2, dbeta = dbeta0 + s1.  The bn flip moves act' (ReLU: a bn flipping across 0 switches it), the
    sigmoid error adds |dz| (1 + |bn|) SIG_ABS (|d silu' / d sigmoid| <= 1 + |bn|); both are carried in *_fl."""
    C = y.shape[-1]
    xh, bn, bfl, xfl = _bn(y, mr, gamma, beta, pre_bias)
    R = xh.shape[0]
    d = dz.to(F64).reshape(-1, C)
    ag = _act_grad(bn, act)
    dev = torch.maximum((_act_grad(bn + bfl, act) - ag).abs(), (_act_grad(bn - bfl, act) - ag).abs())
    dbn = d * ag
    dbn_fl = d.abs() * dev + (d.abs() * (1 + bn.abs()) * SIG_ABS if act == BN_ACT_SILU else 0)
    s1, s2 = dbn.sum(0), (dbn * xh).sum(0)
    s1m, s2m = dbn.abs().sum(0), (dbn * xh).abs().sum(0)
    s1f, s2f = dbn_fl.sum(0), (dbn_fl * xh.abs() + dbn.abs() * xfl).sum(0)
    gd, rs = gamma.to(F64), mr[1].to(F64)
    k = (gd * rs).abs()
    dy = gd * rs * (dbn - s1 / R - xh * s2 / R)
    dy_mag = k * (dbn.abs() + s1m / R + xh.abs() * s2m / R)
    dy_fl = k * (dbn_fl + s1f / R + xh.abs() * s2f / R + xfl * (s2.abs() / R))
    dg0, db0 = dgamma_acc.to(F64), dbeta_acc.to(F64)
    return Result(dy=dy.reshape(y.shape), dy_mag=dy_mag.reshape(y.shape), dy_fl=dy_fl.reshape(y.shape),
                  dgamma=dg0 + s2, dgamma_mag=dg0.abs() + s2m, dgamma_fl=s2f,
                  dbeta=db0 + s1, dbeta_mag=db0.abs() + s1m, dbeta_fl=s1f)


# ---------------------------------------------------------------------------------------------- first conv (Cin = 1)
def conv3x3_c1_fwd(x, w, stride):
    """x [B, T, F], w [Cout, 3, 3] -> (y [B, To, Fo, Cout], magnitude): gemm64.conv3x3_fwd with one input channel."""
    return _g64.conv3x3_fwd(x[..., None], w.reshape(w.shape[0], 3, 3, 1), stride)


def conv3x3_c1_wgrad(dy, x, stride, dw0=None):
    dw, mag = _g64.conv3x3_wgrad(dy, x[..., None], stride, None if dw0 is None else dw0.reshape(dw0.shape[0], 3, 3, 1))
    return dw.reshape(dw.shape[0], 3, 3), mag.reshape(mag.shape[0], 3, 3)


# -------------------------------------------------------------------------------------------------------------- optimizer
def sumsq(g):
    gd = g.to(F64)
    s = (gd * gd).sum()
    return Result(out=s, out_mag=s)


def pow_err(beta, step):
    """Bound on |(1 - powf(fp32(beta), step)) - (1 - beta^step)|: the fp32 beta moves beta^step by
    step |fp32(beta) - beta| / beta of itself, powf adds 2 ulp, and 1 - x one more rounding."""
    b32 = float(np.float32(beta))
    bs = beta ** step
    return bs * (step * abs(b32 - beta) / beta + 4 * U32) + 2 * U32


def adam_step(p32, m, v, g, lr, beta1, beta2, eps, weight_decay, step, sumsq_val, denom=1.0, clip_norm=0.0):
    """fairseq Adam.step after FP16Optimizer's multiply_grads(1 / denom) and clip_grad_norm_(clip_norm):
      gnorm = sqrt(sumsq) / denom;  coef = min(1, clip / (gnorm + 1e-6)) when clip > 0;  g' = g coef / denom (0 at denom 0);
      m = b1 m + (1 - b1) g';  v = b2 v + (1 - b2) g'^2;  step_size = lr sqrt(1 - b2^step) / (1 - b1^step) in doubles;
      p = p - wd lr p;  p = p - step_size m / (sqrt(v) + eps).
    The moment updates take the betas as the fp32 values the kernel receives (1 - fp32(0.999) is 1.3e-5 away from
    0.001, where fairseq's fp32 addcmul_ uses fp32(1 - beta2)); the bias corrections are stated in doubles.
    Bounds: m, v relative to their magnitudes; p to |p (1 - wd lr)| + step_size |m|_mag / (sqrt(v) + eps) plus |u| sz_rel,
    u the update and sz_rel the relative error of the fp32 powf step size (pow_err)."""
    pd, md, vd, gd = p32.to(F64), m.to(F64), v.to(F64), g.to(F64).reshape(-1)[:p32.numel()]
    gscale = 1.0 / denom if denom > 0 else 0.0
    gnorm = math.sqrt(float(sumsq_val)) * gscale
    coef = min(1.0, clip_norm / (gnorm + 1e-6)) if clip_norm > 0 else 1.0
    gi = gd * (gscale * coef)
    b1f, b2f = float(np.float32(beta1)), float(np.float32(beta2))
    m1 = b1f * md + (1 - b1f) * gi
    v1 = b2f * vd + (1 - b2f) * gi * gi
    b1c, b2c = 1 - beta1 ** step, 1 - beta2 ** step
    step_size = lr * math.sqrt(b2c) / b1c
    sz_rel = pow_err(beta1, step) / b1c + 0.5 * pow_err(beta2, step) / b2c
    p1 = pd - weight_decay * lr * pd if weight_decay != 0 else pd
    den = torch.sqrt(v1) + eps
    u = step_size * m1 / den
    p2 = p1 - u
    m_mag = b1f * md.abs() + (1 - b1f) * gi.abs()
    return Result(p=p2, p_mag=p1.abs() + step_size * m_mag / den, p_fl=u.abs() * sz_rel, m=m1,
                  m_mag=m_mag, v=v1, v_mag=b2f * vd.abs() + (1 - b2f) * gi * gi,
                  gnorm=gnorm, coef=coef)
