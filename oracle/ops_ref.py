"""Oracle: plain-PyTorch (CPU, fp32 math) statement of every op in espresso_b200/ops.py, same signatures.

TEST INFRASTRUCTURE ONLY.  Two uses:
  * GPU parity tests compare each CUDA kernel with the function of the same name here;
  * CPU tests monkeypatch these in for `espresso_b200.ops` to exercise the host-side orchestration
    (forward/backward wiring of the Conformer block, flat-buffer optimizer, trainer) against autograd of
    oracle/conformer.py -- no GPU needed.  The product never imports this module.
Each function names the reference computation it restates (see the kernel headers for file:line).
Dropout draws the kernels' own counter-RNG masks (oracle/dropout_rng.py) at the logical element index each kernel
uses, including the device-resident seed installed with set_seed_tensor, so every op is stated at any p.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import dropout_rng as _rng

ACT_NONE, ACT_RELU, ACT_SILU, ACT_RELU_BWD, ACT_SILU_BWD = 0, 1, 2, 3, 4
BF = torch.bfloat16


def _silu_grad(u):
    s = torch.sigmoid(u)
    return s * (1 + u * (1 - s))


# device-resident seed increment (mirror of espresso_b200.ops.set_seed_tensor): added to every op's seed
_SEED_T = None


def set_seed_tensor(t):
    global _SEED_T
    _SEED_T = t


def _keep(seed, idx, p):
    """Keep mask of the logical indices idx (int64 tensor) under the op's seed plus the device seed."""
    dev_seed = 0 if _SEED_T is None else int(_SEED_T.reshape(-1)[0].item())
    return _rng.keep_mask(_rng.combine_seed(seed, dev_seed), idx, p)


def _dscale(p, scale=1.0):
    """The kernels' fp32 rescale of kept elements: scale * 65536 / (65536 - thresh) (just `scale` when p == 0)."""
    if not p > 0:
        return float(np.float32(scale))
    return float(np.float32(np.float32(scale) * np.float32(65536.0)) / np.float32(65536.0 - _rng.thresh(p)))


def _drop(v, p, seed, idx, scale=1.0):
    """fp32 dropout of v with the mask of indices idx: kept elements * _dscale(p, scale), dropped ones 0."""
    v = v * _dscale(p, scale)
    return torch.where(_keep(seed, idx, p), v, torch.zeros_like(v)) if p > 0 else v


def _flat_index(*shape):
    return torch.arange(int(np.prod(shape)), dtype=torch.int64).view(*shape)


def _view(t, nb2, nb1, rows, cols, s2, s1, ld, kmajor):
    """Logical [nb2, nb1, rows, cols] view of a strided operand (cols is the reduction/N dim)."""
    stride = (s2, s1, ld, 1) if kmajor else (s2, s1, 1, ld)
    return t.as_strided((nb2, nb1, rows, cols), stride)


def gemm(A, B, C_out, M, N, K, lda, ldb, ldc, *, a_kmajor=True, b_kmajor=True, nb1=1, nb2=1, sA=(0, 0), sB=(0, 0),
         sC=(0, 0), bias=None, act=ACT_NONE, aux=None, ld_aux=0, sAux=(0, 0), R=None, ldr=0, sR=(0, 0), alpha=1.0,
         beta=1.0, C2=None, drop_p=0.0, drop_mode=0, seed=0, skew_r=0, tile_n=0, accumulate=False, rowsum_a=None,
         rowsum_scale=1.0):
    a = _view(A, nb2, nb1, M, K, sA[1], sA[0], lda, a_kmajor).float()
    b = _view(B, nb2, nb1, N, K, sB[1], sB[0], ldb, b_kmajor).float()
    v = a @ b.transpose(-1, -2)
    if rowsum_a is not None:
        rowsum_a[:M] += rowsum_scale * a.sum(dim=(0, 1, 3))
    if accumulate:
        cv = _view(C_out, nb2, nb1, M, N, sC[1], sC[0], ldc, True)
        cv += (alpha * v).to(C_out.dtype)
        return C_out
    if bias is not None:
        v = v + bias.float()[:N]
    if C2 is not None:
        _view(C2, nb2, nb1, M, N, sC[1], sC[0], ldc, True).copy_(v.to(C2.dtype))
    # epilogue dropout: logical index (bt * M + m) * N + n with bt = b2 * nb1 + b1 (csrc/gemm_tcgen05.cu)
    drop_idx = _flat_index(nb2, nb1, M, N) if drop_mode in (1, 2) else None
    if drop_mode == 2:
        v = _drop(v, drop_p, seed, drop_idx)
    if act == ACT_RELU:
        v = torch.relu(v)
    elif act == ACT_SILU:
        v = F.silu(v)
    elif act in (ACT_RELU_BWD, ACT_SILU_BWD):
        u = _view(aux, nb2, nb1, M, N, sAux[1], sAux[0], ld_aux, True).float()
        v = v * ((u > 0).float() if act == ACT_RELU_BWD else _silu_grad(u))
    if drop_mode == 1:
        v = _drop(v, drop_p, seed, drop_idx)
    v = v * alpha
    if R is not None:
        if skew_r:
            T = skew_r
            full = _view(R, nb2, nb1, M, 2 * T - 1, sR[1], sR[0], ldr, True).float()
            i = torch.arange(M)[:, None]
            j = torch.arange(N)[None, :]
            idx = ((T - 1) - i + j).expand(nb2, nb1, M, N)
            v = v + beta * full.gather(-1, idx)
        else:
            v = v + beta * _view(R, nb2, nb1, M, N, sR[1], sR[0], ldr, True).float()
    _view(C_out, nb2, nb1, M, N, sC[1], sC[0], ldc, True).copy_(v.to(C_out.dtype))
    return C_out


def linear(x, W, bias=None, *, act=ACT_NONE, out=None, out_dtype=BF, **kw):
    M, K = x.shape
    N = W.shape[0]
    if out is None:
        out = torch.empty(M, N, dtype=out_dtype)
    return gemm(x, W, out, M, N, K, x.stride(0), W.stride(0), out.stride(0), bias=bias, act=act, **kw)


def layer_norm_fwd(x, gamma, beta, eps=1e-5, lens=None, T=0, drop_p=0.0, seed=0):
    """Dropout of the output at index r * d + c."""
    xf = x.float()
    mean = xf.mean(-1)
    var = ((xf - mean[:, None]) ** 2).mean(-1)
    rstd = torch.rsqrt(var + eps)
    y = (xf - mean[:, None]) * rstd[:, None] * gamma.float() + beta.float()
    y = _drop(y, drop_p, seed, _rng.row_major_index(*x.shape))
    if lens is not None:
        t = torch.arange(x.shape[0]) % T
        b = torch.arange(x.shape[0]) // T
        y = y * (t < lens[b]).float()[:, None]
    return y.to(BF), mean, rstd


def layer_norm_bwd(dy, x, mean, rstd, gamma, dgamma_acc, dbeta_acc, dres=None, lens=None, T=0, drop_p=0.0, seed=0, next_drop=None):
    """dy is masked with the forward's dropout (index r * d + c); next_drop = (p, seed, scale) adds
    dropout(bf16 dx) * scale on the same index as a second output."""
    dyf = dy.float()
    if lens is not None:
        t = torch.arange(x.shape[0]) % T
        b = torch.arange(x.shape[0]) // T
        dyf = dyf * (t < lens[b]).float()[:, None]
    dyf = _drop(dyf, drop_p, seed, _rng.row_major_index(*x.shape))
    xh = (x.float() - mean[:, None]) * rstd[:, None]
    g = dyf * gamma.float()
    dx = rstd[:, None] * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    if dres is not None:
        dx = dx + dres.float()
    dgamma_acc += (dyf * xh).sum(0)
    dbeta_acc += dyf.sum(0)
    if next_drop is not None:
        return dx.to(BF), dropout(dx.to(BF), next_drop[0], next_drop[1], scale=next_drop[2])
    return dx.to(BF)


def colsum(x, out_acc, scale=1.0):
    out_acc += scale * x.float().sum(0)


def dropout(x, p, seed, scale=1.0, out=None):
    """Index r * N + c with N the logical number of columns (not the row stride of x)."""
    y = _drop(x.float(), p, seed, _rng.row_major_index(*x.shape), scale).to(BF)
    if out is not None:
        out.copy_(y)
        return out
    return y


def mask_rows_(x, lens):
    B, T, _ = x.shape
    x *= (torch.arange(T)[None, :] < lens[:, None]).to(x.dtype)[:, :, None]
    return x


def qprep_fwd(q, u, v, scale):
    qf = q.float()
    qu = ((qf + u.float()).to(BF).float() * scale).to(BF)
    qv = ((qf + v.float()).to(BF).float() * scale).to(BF)
    return qu, qv


def qprep_bwd(dqu, dqv, scale, dq_out):
    dq_out.copy_((scale * (dqu.float() + dqv.float())).to(BF))


def attn_softmax_fwd(scores, T, lens, drop_p=0.0, seed=0, causal=False):
    """Dropout of the probabilities at index row * ld + j, row = (h * B + b) * Tq + i."""
    H, B, Tq, ld = scores.shape
    s = scores.float()[..., :T].clone()
    if lens is not None:
        km = torch.arange(T)[None, :] >= lens[:, None]  # [B, T] keys to mask
        s = s.masked_fill(km[None, :, None, :], float("-inf"))
    if causal:
        fut = torch.arange(T)[None, :] > torch.arange(Tq)[:, None]
        s = s.masked_fill(fut[None, None], float("-inf"))
    p = torch.zeros(H, B, Tq, ld)
    p[..., :T] = torch.softmax(s, dim=-1)
    p = p.to(BF)
    if drop_p > 0:
        return p, _drop(p.float(), drop_p, seed, _flat_index(H, B, Tq, ld)).to(BF)
    return p, p


def attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens, drop_p=0.0, seed=0, save_probs=True, pos_hstride=None, key_bounds=None):
    """fairseq/modules/multihead_attention.py:788-897 (rel-pos branch) in fp32: AC + skew(BD), key-padding mask, softmax,
    P v.  Same return convention as espresso_b200.ops.attn_fused_fwd; dropout at index row * ld + j
    as in attn_softmax_fwd."""
    R, d = qu.shape
    hd = d // H
    if pos_hstride is None:
        pos_hstride = hd if pos.shape[1] == d else 0
    quh = qu.float().view(B, T, H, hd).permute(2, 0, 1, 3)                    # [H, B, T, hd]
    qvh = qv.float().view(B, T, H, hd).permute(2, 0, 1, 3)
    kh = k.float().reshape(B, T, H, hd).permute(2, 0, 1, 3)
    vh = v.float().reshape(B, T, H, hd).permute(2, 0, 1, 3)
    ph = torch.stack([pos.float()[:, h * pos_hstride: h * pos_hstride + hd] for h in range(H)])   # [H, 2T-1, hd]
    ac = quh @ kh.transpose(-1, -2)
    bd_full = (qvh @ ph[:, None].transpose(-1, -2)).to(BF).float()           # the reference keeps BD in the model dtype
    i = torch.arange(T)[:, None]
    j = torch.arange(T)[None, :]
    s = ac + bd_full.gather(-1, ((T - 1) - i + j).expand(H, B, T, T))
    if key_bounds is not None:   # attn_mask: bf16(-1e4) ADDED on the hidden keys in the model dtype
        lo, hi = key_bounds      # (transformer_layer.py:189-192, multihead_attention.py:835-839)
        hidden = (j < lo.long()[:, None]) | (j >= hi.long()[:, None])
        s = torch.where(hidden.expand_as(s), (s - 9984.0).to(BF).float(), s)
    if lens is not None:
        km = torch.arange(T)[None, :] >= lens[:, None]
        s = s.masked_fill(km[None, :, None, :], float("-inf"))
    pr = torch.softmax(s, dim=-1).to(BF)
    ld = (T + 7) // 8 * 8
    prd = pr
    if drop_p > 0:
        prd = _drop(pr.float(), drop_p, seed, _flat_index(H, B, T, ld)[..., :T]).to(BF)
    ctx = (prd.float() @ vh).permute(1, 2, 0, 3).reshape(R, d).to(BF)
    p = pd = None
    if save_probs:
        p = torch.zeros(H, B, T, ld, dtype=BF)
        p[..., :T] = pr
        pd = p
        if drop_p > 0:
            pd = torch.zeros(H, B, T, ld, dtype=BF)
            pd[..., :T] = prd
    return ctx, p, pd


def attn_fused_bwd(dctx, ctx, qu, v, p, pd, B, T, H, ldp, dk_out, dv_out, drop_p=0.0, seed=0):
    """The unfused chain in fp32: dPd = dctx v^T, softmax backward (+ skewed copy), dV = P_drop^T dctx, dK = dS^T qu."""
    R, d = dctx.shape
    hd = d // H
    dh = dctx.float().view(B, T, H, hd).permute(2, 0, 1, 3)                    # [H, B, T, hd]
    vh = v.float().reshape(B, T, H, hd).permute(2, 0, 1, 3)
    quh = qu.float().view(B, T, H, hd).permute(2, 0, 1, 3)
    ld = p.shape[-1]
    dpd = torch.zeros(H, B, T, ld)
    dpd[..., :T] = dh @ vh.transpose(-1, -2)
    ds, dbd = attn_softmax_bwd(p, dpd, T, ldp, drop_p, seed)
    dv = pd.float()[..., :T].transpose(-1, -2) @ dh                            # [H, B, T, hd]
    dk = ds.float()[..., :T].transpose(-1, -2) @ quh
    dv_out.copy_(dv.permute(1, 2, 0, 3).reshape(R, d).to(BF))
    dk_out.copy_(dk.permute(1, 2, 0, 3).reshape(R, d).to(BF))
    return ds, dbd


def attn_softmax_bwd(p, dp_drop, T, ldp, drop_p=0.0, seed=0, want_dbd=True):
    H, B, Tq, ld = p.shape
    pf = p.float()[..., :T]
    dp = _drop(dp_drop.float(), drop_p, seed, _flat_index(H, B, Tq, ld))[..., :T]
    ds_ = pf * (dp - (dp * pf).sum(-1, keepdim=True))
    ds = torch.zeros(H, B, Tq, ld)
    ds[..., :T] = ds_
    ds = ds.to(BF)
    dbd = None
    if want_dbd:
        dbd = torch.zeros(H, B, T, ldp)
        i = torch.arange(T)[:, None]
        j = torch.arange(T)[None, :]
        idx = ((T - 1) - i + j).expand(H, B, T, T)
        dbd.scatter_(-1, idx, ds[..., :T].float())
        dbd = dbd.to(BF)
    return ds, dbd


def _glu(g):
    C = g.shape[-1] // 2
    return (g[..., :C].float() * torch.sigmoid(g[..., C:].float())).to(BF).float()


def glu_dwconv_fwd(g, w):
    B, T, C2 = g.shape
    C, k = w.shape
    gl = _glu(g).transpose(1, 2)  # [B, C, T]
    y = F.conv1d(gl, w.float()[:, None, :], padding=k // 2, groups=C).transpose(1, 2).contiguous().to(BF)
    yf = y.double().reshape(-1, C)
    stats = torch.stack([yf.sum(0), (yf * yf).sum(0)])
    return y, stats


def glu_dwconv_bwd(dy, g, w, dw_acc):
    B, T, C2 = g.shape
    C, k = w.shape
    with torch.enable_grad():  # may be called from inside an autograd.Function.backward
        a = g[..., :C].float().detach().requires_grad_(True)
        gate = g[..., C:].float().detach().requires_grad_(True)
        wf = w.float().detach().requires_grad_(True)
        gl = (a * torch.sigmoid(gate))
        y = F.conv1d(gl.transpose(1, 2), wf[:, None, :], padding=k // 2, groups=C).transpose(1, 2)
        y.backward(dy.float())
    dw_acc += wf.grad
    return torch.cat([a.grad, gate.grad], dim=-1).to(BF)


def bn_finalize(stats, R, C_, eps, momentum, run_mean, run_var, training):
    if training:
        m = stats[0] / R
        var = (stats[1] / R - m * m).clamp_min(0)
        mr = torch.stack([m.float(), torch.rsqrt(var.float() + eps)])
        if run_mean is not None:
            unb = var * R / (R - 1) if R > 1 else var
            run_mean.mul_(1 - momentum).add_(momentum * m.float())
            run_var.mul_(1 - momentum).add_(momentum * unb.float())
        return mr
    return torch.stack([run_mean.float(), torch.rsqrt(run_var.float() + eps)])


BN_ACT_SILU, BN_ACT_RELU = 1, 2


def _pre(y, pre_bias):
    """bf16(y + pre_bias[c]): the conv bias folded into the BatchNorm kernels."""
    return y if pre_bias is None else (y.float() + pre_bias.float()).to(BF)


def _conv_nchw(x, w, stride):
    xin = x.float().unsqueeze(1) if x.dim() == 3 else x.float().permute(0, 3, 1, 2)
    wt = w.float().permute(0, 3, 1, 2) if w.dim() == 4 else w.float().reshape(w.shape[0], 1, 3, 3)
    return xin, wt


def conv3x3_fwd(x, w, stride):
    xin, wt = _conv_nchw(x, w, stride)
    return F.conv2d(xin, wt, None, tuple(stride), (1, 1)).permute(0, 2, 3, 1).contiguous().to(BF)


def conv3x3_dgrad(dy, w, in_shape, stride):
    B, T, F_, Cin = in_shape
    wt = w.float().permute(0, 3, 1, 2)
    dx = torch.nn.grad.conv2d_input((B, Cin, T, F_), wt, dy.float().permute(0, 3, 1, 2), tuple(stride), (1, 1))
    return dx.permute(0, 2, 3, 1).contiguous().to(BF)


def conv3x3_wgrad(dy, x, dw_acc, stride):
    xin, _ = _conv_nchw(x, dw_acc, stride)
    Cout, Cin = dy.shape[-1], xin.shape[1]
    dw = torch.nn.grad.conv2d_weight(xin, (Cout, Cin, 3, 3), dy.float().permute(0, 3, 1, 2), tuple(stride), (1, 1))
    dw_acc += dw.permute(0, 2, 3, 1).reshape(dw_acc.shape)


def bn_stats(x, C_, pre_bias=None):
    x = _pre(x, pre_bias)
    xf = x.double().reshape(-1, C_)
    return torch.stack([xf.sum(0), (xf * xf).sum(0)])


def bn_act_fwd(y, mr, gamma, beta, act=BN_ACT_SILU, pre_bias=None):
    y = _pre(y, pre_bias)
    bn = ((y.float() - mr[0]) * mr[1] * gamma.float() + beta.float()).to(BF).float()
    return (F.silu(bn) if act == BN_ACT_SILU else torch.relu(bn)).to(BF)


def bn_act_bwd(dz, y, mr, gamma, beta, dgamma_acc, dbeta_acc, act=BN_ACT_SILU, pre_bias=None):
    y = _pre(y, pre_bias)
    Cn = y.shape[-1]
    yf = y.float().reshape(-1, Cn)
    xh = (yf - mr[0]) * mr[1]
    bn = (xh * gamma.float() + beta.float()).to(BF).float()
    dbn = dz.float().reshape(-1, Cn) * (_silu_grad(bn) if act == BN_ACT_SILU else (bn > 0).float())
    s1, s2 = dbn.sum(0), (dbn * xh).sum(0)
    n = yf.shape[0]
    dy = gamma.float() * mr[1] * (dbn - s1 / n - xh * s2 / n)
    dgamma_acc += s2
    dbeta_acc += s1
    return dy.to(BF).reshape(y.shape)


def bn_silu_fwd(y, mr, gamma, beta):
    return bn_act_fwd(y, mr, gamma, beta, BN_ACT_SILU)


def bn_silu_bwd(dz, y, mr, gamma, beta, dgamma_acc, dbeta_acc):
    return bn_act_bwd(dz, y, mr, gamma, beta, dgamma_acc, dbeta_acc, BN_ACT_SILU)


def sumsq(g, out):
    out.copy_((g.double() ** 2).sum().float().reshape(out.shape))
    return out


def adam_step(p32, m, v, g, p16, lr, beta1, beta2, eps, weight_decay, step, sumsq_t, denom_dev=None, denom_const=1.0,
              clip_norm=0.0, gnorm_out=None, hyper_dev=None):
    n = p32.numel()
    if hyper_dev is not None:
        lr, step = float(hyper_dev[0]), float(hyper_dev[1])
    denom = float(denom_dev.item()) if denom_dev is not None else denom_const
    gscale = 1.0 / denom if denom > 0 else 0.0
    gnorm = float(sumsq_t.item()) ** 0.5 * gscale
    coef = min(1.0, clip_norm / (gnorm + 1e-6)) if clip_norm > 0 else 1.0
    if gnorm_out is not None:
        gnorm_out.fill_(gnorm)
    gi = g.view(-1)[:n] * (gscale * coef)
    m.mul_(beta1).add_((1 - beta1) * gi)
    v.mul_(beta2).add_((1 - beta2) * gi * gi)
    b1, b2 = 1 - beta1 ** step, 1 - beta2 ** step
    if weight_decay != 0:
        p32.add_(p32, alpha=-weight_decay * lr)
    p32.addcdiv_(m, v.sqrt() + eps, value=-lr * (b2 ** 0.5) / b1)
    p16.copy_(p32.to(BF))


def cast_f32_bf16(x, y):
    y.copy_(x.to(BF))


def cast_bf16_f32(x, y):
    y.copy_(x.float())


def frontend_fbank(wave, n_samples, cmvn_mean=None, cmvn_std=None, freq_masks=None, time_masks=None, t_max=None,
                   out_dtype=BF, workspace=None):
    import numpy as np

    from oracle import frontend as O

    B = wave.shape[0]
    if t_max is None:
        t_max = O.num_frames(wave.shape[1])
    out = torch.zeros(B, t_max, 80)
    lens = torch.zeros(B, dtype=torch.int32)
    for b in range(B):
        n = int(n_samples[b])
        fb = O.kaldi_fbank(wave[b, :n].float().numpy())
        m = fb.shape[0]
        lens[b] = m
        if m == 0:
            continue
        x = fb.astype(np.float64)
        if cmvn_mean is not None:
            x = O.global_cmvn(fb, cmvn_mean.double().numpy(), cmvn_std.double().numpy())
        fill = x.mean()
        y = x.copy()
        if freq_masks is not None:
            for f0, f in freq_masks[b].tolist():
                if f > 0:
                    y[:, f0:f0 + f] = fill
        if time_masks is not None:
            for t0, t in time_masks[b].tolist():
                if t > 0:
                    y[t0:t0 + t, :] = fill
        out[b, :m] = torch.from_numpy(y).float()
    return out.to(out_dtype), lens


def ctc_loss(logits, V, in_lens, targets, tgt_lens, blank, zero_infinity=True, grad_scale=1.0, want_grad=True):
    from oracle import ctc as O

    B, T, ld = logits.shape
    loss = torch.zeros(B)
    grad = torch.zeros(B, T, ld)
    for b in range(B):
        nll, g = O.ctc_loss_and_grad(logits[b, :, :V].float().numpy(), int(in_lens[b]),
                                     targets[b, : int(tgt_lens[b])].numpy(), blank, zero_infinity)
        loss[b] = float(nll)
        grad[b, :, :V] = torch.from_numpy(g).float() * grad_scale
    return loss, (grad.to(BF) if want_grad else None)


SMOOTH_UNIFORM, SMOOTH_UNIGRAM, SMOOTH_TEMPORAL = 0, 1, 2


def smoothing_weights(V, targets, pad_idx, eps, smoothing=SMOOTH_UNIFORM, unigram=None, U=0):
    """(a, w [R, V]) with loss = a * nll + sum_v w_v * (-lprobs_v)
    (espresso/criterions/label_smoothed_cross_entropy_v2.py:49-79 temporal mask, :95-119 combination)."""
    t = targets.long()
    R = t.numel()
    if smoothing == SMOOTH_UNIFORM:
        eps_i = eps / (V - 1)
        return 1 - eps - eps_i, torch.full((R, V), eps_i)
    if smoothing == SMOOTH_UNIGRAM:
        return 1 - eps, (eps * unigram.float()[:V])[None, :].expand(R, V)
    tt = t.view(-1, U)
    m = torch.zeros(tt.shape[0], U, V)
    for off, c in ((-2, 2.0), (-1, 5.0), (1, 5.0), (2, 2.0)):
        src = torch.full_like(tt, pad_idx)
        if off < 0:
            src[:, -off:] = tt[:, :off]
        else:
            src[:, :-off] = tt[:, off:]
        m.scatter_add_(-1, src[:, :, None], torch.full((tt.shape[0], U, 1), c))
    m[:, :, pad_idx] = 0
    tot = m.sum(-1, keepdim=True)
    tot[tot == 0] = 1.0
    return 1 - eps, eps * (m / tot).view(R, V)


def lsce_loss(logits, V, targets, pad_idx, eps, grad_scale=1.0, want_grad=True, smoothing=SMOOTH_UNIFORM, unigram=None, U=0):
    x = logits.float()[:, :V]
    lp = torch.log_softmax(x, dim=-1)
    t = targets.long()
    nll = -lp.gather(1, t[:, None]).squeeze(1)
    a, w = smoothing_weights(V, targets, pad_idx, eps, smoothing, unigram, U)
    keep = (t != pad_idx).float()
    loss = (a * nll - (w * lp).sum(-1)) * keep
    grad = None
    if want_grad:
        g = torch.softmax(x, dim=-1) * (a + w.sum(-1, keepdim=True)) - w
        g[torch.arange(x.shape[0]), t] -= a
        grad = torch.zeros_like(logits, dtype=torch.float32)
        grad[:, :V] = g * keep[:, None] * grad_scale
        grad = grad.to(BF)
    return loss, nll * keep, grad


def embed_fwd(tokens, E, pos, U, scale, pad_idx, drop_p=0.0, seed=0):
    """Dropout at index r * d + c (csrc/lsce.cu embed_fwd_kernel)."""
    t = tokens.long()
    x = (E[t].float() * scale).to(BF).float()
    if pos is not None:
        pidx = torch.arange(t.numel()) % U
        x = x + pos[pidx].float() * (t != pad_idx).float()[:, None]
    return _drop(x, drop_p, seed, _rng.row_major_index(*x.shape)).to(BF)


def embed_bwd(tokens, dx, dE_acc, scale, pad_idx, drop_p=0.0, seed=0):
    """dE[tok] += dropout(dx) * scale, mask index r * d + c; pad rows get nothing."""
    t = tokens.long()
    keep = (t != pad_idx)
    g = _drop(dx.float(), drop_p, seed, _rng.row_major_index(*dx.shape), scale)
    dE_acc.index_add_(0, t[keep], g[keep])


def argmax_rows(x, V):
    return x[:, :V].float().argmax(-1).to(torch.int32)


def beam_merge(x, V, x_is_logits, out, prev_scores=None, temperature=1.0, lm=None, lm_is_logits=True, lm_weight=0.0,
               pad=1, unk=3, unk_penalty=0.0, eos=2, force_eos=False, eos_factor=None, ban_eos=False):
    lp = x.float()[:, :V]
    if x_is_logits:
        lp = torch.log_softmax(lp / temperature, dim=-1)
    lp = lp.clone()
    if lm is not None:
        l = lm.float()[:, :V]
        lp += lm_weight * (torch.log_softmax(l, dim=-1) if lm_is_logits else l)
    lp[lp != lp] = float("-inf")
    lp[:, pad] = float("-inf")
    lp[:, unk] -= unk_penalty
    if force_eos:
        lp[:, :eos] = float("-inf")
        lp[:, eos + 1:] = float("-inf")
    elif eos_factor is not None:
        dis = lp[:, eos] < eos_factor * lp.max(dim=1)[0]
        lp[dis, eos] = float("-inf")
    if ban_eos:
        lp[:, eos] = float("-inf")
    if prev_scores is not None:
        lp = lp + prev_scores[:, None]
    out.copy_(lp)
    return out


def beam_topk(cand, bsz, sent_stride, n_cand, K, V):
    flat = cand.reshape(-1)
    s = torch.empty(bsz, K)
    t = torch.empty(bsz, K, dtype=torch.int32)
    b = torch.empty(bsz, K, dtype=torch.int32)
    for i in range(bsz):
        c = flat[i * sent_stride: i * sent_stride + n_cand]
        order = sorted(range(n_cand), key=lambda j: (-float(c[j]) if c[j] == c[j] else float("inf"), j))[:K]
        for r, j in enumerate(order):
            s[i, r], t[i, r], b[i, r] = c[j], j % V, j // V
    return s, t, b


def beam_bookkeep(step, max_len, bsz, beam, K, eos, pad, normalize, len_penalty, cs, ct, cb, st):
    NEG = float("-inf")
    L = max_len + 2
    tin, sin = st.tokens, st.scores
    tout, sout = st.tokens_alt, st.scores_alt
    for s in range(bsz):
        rb = s * beam
        if st.finished[s]:
            tout[rb:rb + beam] = tin[rb:rb + beam]
            sout[rb:rb + beam] = sin[rb:rb + beam]
            st.new_order[rb:rb + beam] = torch.arange(rb, rb + beam, dtype=torch.int32)
            continue
        had_eos = False
        for c in range(min(beam, K)):
            if int(ct[s, c]) == eos and float(cs[s, c]) != NEG and not st.ignore[rb + c]:
                had_eos = True
                slot = int(st.nfin[s])
                if slot < beam:
                    row = rb + int(cb[s, c])
                    st.fin_tokens[s, slot, :step] = tin[row, 1:step + 1]
                    st.fin_tokens[s, slot, step] = eos
                    cum = torch.cat([sin[row, :step], cs[s, c].reshape(1)])
                    pos = cum.clone()
                    pos[1:] = cum[1:] - cum[:-1]
                    st.fin_pos[s, slot, :step + 1] = pos
                    st.fin_len[s, slot] = step + 1
                    st.fin_score[s, slot] = cs[s, c] / (step + 1) ** len_penalty if normalize else cs[s, c]
                    st.nfin[s] = slot + 1
        done = False
        if had_eos and (int(st.nfin[s]) == beam or step == max_len):
            st.finished[s] = 1
            st.n_unfinished -= 1
            done = True
        if done or step >= max_len:
            tout[rb:rb + beam] = tin[rb:rb + beam]
            sout[rb:rb + beam] = sin[rb:rb + beam]
            st.new_order[rb:rb + beam] = torch.arange(rb, rb + beam, dtype=torch.int32)
            continue
        chosen = []
        for want_masked in (False, True):
            for c in range(K):
                raw = int(ct[s, c]) == eos and float(cs[s, c]) != NEG
                masked = (raw or bool(st.ignore[rb + c])) if c < beam else raw
                if masked == want_masked and len(chosen) < beam:
                    chosen.append((c, masked))
        while len(chosen) < beam:
            chosen.append((0, True))
        for k, (c, masked) in enumerate(chosen):
            old = rb + int(cb[s, c])
            tout[rb + k, :step + 1] = tin[old, :step + 1]
            tout[rb + k, step + 1] = ct[s, c]
            tout[rb + k, step + 2:] = pad
            sout[rb + k, :step] = sin[old, :step]
            sout[rb + k, step] = cs[s, c]
            st.new_order[rb + k] = old
        for k, (c, masked) in enumerate(chosen):
            st.ignore[rb + k] = 1 if masked else 0
    st.tokens, st.tokens_alt = tout, tin
    st.scores, st.scores_alt = sout, sin


def gather_rows(src, idx, out=None):
    r = src[idx.long()]
    if out is not None:
        out.copy_(r)
        return out
    return r


def decode_self_attn(q, kv_cache, anc, T, H, scale):
    N, d = q.shape
    hd = d // H
    rows = anc[:T].long()                                   # [T, N]
    kvs = kv_cache[:T].float()[torch.arange(T)[:, None], rows]  # [T, N, 2d]
    k = kvs[..., :d].reshape(T, N, H, hd)
    v = kvs[..., d:].reshape(T, N, H, hd)
    qh = q.float().reshape(N, H, hd)
    s = torch.einsum("nhc,tnhc->nht", qh, k) * scale
    p = torch.softmax(s, dim=-1).to(BF).float()
    return torch.einsum("nht,tnhc->nhc", p, v).reshape(N, d).to(BF)


def decode_cross_attn(q, kv, lens, beam, H, scale):
    N, d = q.shape
    hd = d // H
    bsz, Tk, _ = kv.shape
    sent = torch.arange(N) // beam
    k = kv.float()[sent][..., :d].reshape(N, Tk, H, hd)
    v = kv.float()[sent][..., d:].reshape(N, Tk, H, hd)
    s = torch.einsum("nhc,nthc->nht", q.float().reshape(N, H, hd), k) * scale
    if lens is not None:
        mask = torch.arange(Tk)[None, :] >= lens[sent][:, None]
        s = s.masked_fill(mask[:, None, :], float("-inf"))
    p = torch.softmax(s, dim=-1).to(BF).float()
    return torch.einsum("nht,nthc->nhc", p, v).reshape(N, d).to(BF)


def decode_update_ancestry(anc_in, anc_out, new_order, step):
    N = anc_in.shape[1]
    if step > 0:
        src = anc_in[:step]
        anc_out[:step] = src[:, new_order.long()] if new_order is not None else src
    anc_out[step] = torch.arange(N, dtype=anc_out.dtype)


def joint_fwd(enc, dec):
    return torch.relu(enc.float()[:, :, None, :] + dec.float()[:, None, :, :]).to(BF)


def joint_bwd(df, f):
    g = df.float() * (f.float() > 0).float()
    return g.sum(2).to(BF), g.sum(1)


def rnnt_loss(logits, V, t_lens, u_lens, targets, blank, grad_scale=1.0, want_grad=True):
    """Oracle: the reference's own call -- torchaudio.functional.rnnt_loss with fused log-softmax, clamp=-1
    (espresso/criterions/transducer_loss.py:130-140), differentiated by autograd, on fp32 copies of the bf16 logits."""
    import torchaudio

    with torch.enable_grad():
        x = logits.detach().float()[..., :V].clone().requires_grad_(True)
        loss = torchaudio.functional.rnnt_loss(x, targets.int(), t_lens.int(), u_lens.int(), blank=blank, clamp=-1.0, reduction="none")
        grad = None
        if want_grad:
            loss.sum().backward()
            grad = torch.zeros_like(logits, dtype=torch.float32)
            grad[..., :V] = x.grad * grad_scale
            grad = grad.to(BF)
    return loss.detach(), grad


# ---- look-ahead word-LM fusion (csrc/lookahead.cu): same call signatures as espresso_b200.ops ---------------------------
def lookahead_words(nodes_in, new_order, node_word, word_unk, nodes_out, words):
    n = nodes_in if new_order is None else nodes_in[new_order.long()]
    w = node_word[n.long()]
    nodes_out.copy_(n)
    words.copy_(torch.where(w < 0, torch.full_like(w, word_unk), w))


def wordlm_cumsum(logits, Vw, prev_tokens, tok_stride, space_idx, first, cum_in, new_order, cum_out, eos_logprob, word_eos,
                  log_mode=False):
    x = logits[:, :Vw].double()
    lp = torch.log_softmax(x, -1)
    new = lp.float() if log_mode else lp.exp().cumsum(-1).float()
    if first:
        cum_out.copy_(new)
    else:
        old = cum_in if new_order is None else cum_in[new_order.long()]
        cum_out.copy_(torch.where((prev_tokens == space_idx)[:, None], new, old))
    eos_logprob.copy_(lp[:, word_eos].float())


def lookahead_step(prev_tokens, tok_stride, first, nodes_in, nodes_out, cum, Vw, eos_logprob, tree, space_idx, eos_idx, pad_idx,
                   word_unk, oov_penalty, open_vocab, zero, out, Vs):
    """espresso/models/tensorized_lookahead_language_model.py:150-263 on the CSR tree, one hypothesis at a time."""
    off, tok, child = tree["child_off"].tolist(), tree["child_tok"].tolist(), tree["child_node"].tolist()
    word, lo, hi = tree["node_word"].tolist(), tree["node_lo"].tolist(), tree["node_hi"].tolist()
    cs_all = cum.double()
    out.fill_(float("-inf"))
    for n in range(nodes_in.numel()):
        prev = int(prev_tokens[n])
        after_space = (not first) and prev == space_idx
        if first or after_space:
            node = 1
        else:
            cur, node = int(nodes_in[n]), 0
            for e in range(off[cur], off[cur + 1]):
                if tok[e] == prev:
                    node = child[e]
        nodes_out[n] = node
        cs = cs_all[n]
        if not open_vocab:
            row = torch.full((Vs,), zero, dtype=torch.float64)
        elif node == 0:
            row = torch.ones(Vs, dtype=torch.float64)
        else:
            row = torch.full((Vs,), float(oov_penalty * (cs[word_unk] - cs[word_unk - 1])), dtype=torch.float64)
            if after_space or prev == eos_idx:
                row[space_idx] = zero
            if not after_space:
                row[eos_idx] = zero
        sum_p = float(cs[hi[node]] - cs[lo[node]]) if node > 1 else 1.0
        for e in range(off[node], off[node + 1]):
            c = child[e]
            row[tok[e]] = zero if sum_p < zero else float(cs[hi[c]] - cs[lo[c]]) / sum_p
        row[pad_idx] = zero
        if word[node] >= 0:
            row[space_idx] = zero if sum_p < zero else float(cs[word[node]] - cs[word[node] - 1]) / sum_p
        lp = row.clamp(min=zero).log().float()
        if after_space:
            lp[eos_idx] = eos_logprob[n]
        out[n, :Vs] = lp


def multilevel_step(prev_tokens, tok_stride, first, nodes_in, nodes_out, new_order, wlp, Vw, sub, sub_is_logits, sub_weight, out_prev,
                    cumlp_in, cumlp_out, tree, space_idx, eos_idx, word_unk, word_eos, log_oov_penalty, open_vocab, logzero, out, Vs):
    """espresso/models/external_language_model.py:437-533 on the CSR tree."""
    off, tok, child, word = (tree[k].tolist() for k in ("child_off", "child_tok", "child_node", "node_word"))
    rows = torch.log_softmax(sub[:, :Vs].float(), -1) if sub_is_logits else sub[:, :Vs].float()
    out.fill_(float("-inf"))
    for n in range(nodes_in.numel()):
        prev = int(prev_tokens[n])
        after_space = (not first) and prev == space_idx
        src = n if new_order is None else int(new_order[n])
        if first or after_space:
            node = 1
        else:
            cur, node = int(nodes_in[n]), 0
            for e in range(off[cur], off[cur + 1]):
                if tok[e] == prev:
                    node = child[e]
        is_child = (not first) and (not after_space) and node != 0
        cum = 0.0
        if not first and ((not after_space) if open_vocab else is_child):
            cum = float(cumlp_in[src]) + float(out_prev[src, prev])
        row = rows[n] * sub_weight
        if (not open_vocab) and (not first) and (not after_space) and (not is_child):
            row = torch.full_like(row, logzero)
        w = word[node]
        v_space = float(wlp[n, w if w >= 0 else word_unk]) + (-cum if w >= 0 else log_oov_penalty)
        if after_space or prev == eos_idx:
            v_space = logzero
        row[space_idx] = v_space
        row[eos_idx] = row[eos_idx] + wlp[n, word_eos] if after_space else logzero
        out[n, :Vs] = row
        nodes_out[n] = node
        cumlp_out[n] = cum
