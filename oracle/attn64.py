"""Float64 references of the attention kernels (csrc/attn_fused.cu, csrc/attn_fused_bwd.cu, the softmax kernels of
csrc/elementwise.cu and csrc/decode_attn.cu), with per-element error bounds.

TEST INFRASTRUCTURE ONLY.  Inputs are the kernels' own bf16 tensors, widened exactly; dropout masks come from
oracle/dropout_rng.py, so they are the kernels' masks bit for bit.  Each reference models the rounding points the kernels
document and nothing else:
  * BD = q_v pos^T is rounded to bf16 before the skew (the reference keeps BD in the model dtype);
  * a key hidden by a key range gets bf16(s - 9984) (bf16(-1e4) added in the model dtype);
  * the probabilities are cast to bf16 before P V (and, with dropout, rescaled in fp32 and cast again);
  * unfused scores are the bf16 output of their GEMM.
Every result comes with the quantities its bound is built from, and bounds read |x - x64| <= bound, as in gemm64:
  logits     e_ij = tau * (|qu_i||k_j| + |qv_i||pos_(T-1)-i+j|) + one bf16 ulp of BD64 (+ of the hidden-key rounding)
  softmax    |dp_ij| <= p_ij * (expm1(2 max_k e_ik) + exp_ij + sum_k p_ik exp_ik + (T + 16) 2^-24)
             (exp_ij: the fp32 exp2 / __expf error, 2^-21 (2 + |s_ij - m_i| + 2 |m_i|))
  bf16 out   |RN(x) - x64| <= (1 + 2^-8) |x - x64| + 2^-8 |x64|
  P V        ctx64 = sum_j Pd64_j v_j, bound sum_j dPd_j |v_j| + tau_acc sum_j Pd64_j |v_j|, then one bf16 rounding.
tau is the fp32 reduction error per unit of magnitude, measured on the GPU (tests/test_gpu_attn_reference.py).
Runs on the device of its inputs.
"""
import numpy as np
import torch

from oracle import dropout_rng as _rng

F64 = torch.float64
BF = torch.bfloat16
U32 = 2.0 ** -24           # fp32 unit roundoff
BF_REL = 2.0 ** -8         # half a bf16 ulp (8 significant bits), relative
BF_ULP = 2.0 ** -7         # one bf16 ulp, relative (upper bound)
EXP_REL = 2.0 ** -21       # ex2.approx / __expf relative error per unit of exponent (with the fma rounding of the argument)
HIDDEN = 9984.0            # bf16(-1e4)


def r8(n):
    return (n + 7) // 8 * 8


def bf16_out(err, x64):
    """Bound of a bf16-rounded output whose unrounded value is within err of x64."""
    return (1 + BF_REL) * err + BF_REL * x64.abs()


def keep_mask(seed, shape, ld_last, p, device, device_seed=0):
    """Dropout keep mask of a [H, B, Tq, n] block of a [H, B, Tq, ld_last] probability tensor (index row * ld + j)."""
    H, B, Tq, n = shape
    rows = torch.arange(H * B * Tq, dtype=torch.int64)[:, None] * ld_last + torch.arange(n, dtype=torch.int64)[None, :]
    k = _rng.keep_mask(_rng.combine_seed(seed, device_seed), rows, p)
    return k.view(H, B, Tq, n).to(device)


def dscale(p):
    return _rng.scale(p)


def heads(x, B, T, H):
    """[B*T, >= H*hd] (any row stride) -> [H, B, T, hd] float64."""
    return x.to(F64).reshape(B, T, H, x.shape[1] // H).permute(2, 0, 1, 3)


def _skew(full, T):
    """BD[..., i, j] = full[..., i, (T-1) - i + j]."""
    i = torch.arange(T, device=full.device)[:, None]
    j = torch.arange(T, device=full.device)[None, :]
    return full.gather(-1, ((T - 1) - i + j).expand(*full.shape[:-1], T))


def unskew(ds, T, ldp):
    """dBD[..., i, (T-1) - i + j] = ds[..., i, j], zeros elsewhere, [..., T, ldp]."""
    out = torch.zeros(*ds.shape[:-1], ldp, dtype=ds.dtype, device=ds.device)
    i = torch.arange(T, device=ds.device)[:, None]
    j = torch.arange(T, device=ds.device)[None, :]
    out.scatter_(-1, ((T - 1) - i + j).expand(*ds.shape[:-1], T), ds[..., :T])
    return out


def softmax64(s, vis, e=None):
    """Softmax over the last axis of float64 logits s at the visible keys (vis); a row without visible keys is 0.
    e: per-logit error bound (or None: exact logits).  Returns (p, bound of the kernel's fp32 p before its bf16 cast)."""
    s = torch.where(vis, s, torch.full_like(s, -float("inf")))
    m = s.amax(-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    z = torch.where(vis, torch.exp(s - m), torch.zeros_like(s))
    l = z.sum(-1, keepdim=True)
    p = torch.where(l > 0, z / torch.where(l > 0, l, torch.ones_like(l)), torch.zeros_like(z))
    T = s.shape[-1]
    rel = torch.where(vis, EXP_REL * (2 + (s - m).abs() + 2 * m.abs()), torch.zeros_like(s))
    coef = rel + (p * rel).sum(-1, keepdim=True) + (T + 16) * U32
    if e is not None:
        E = torch.where(vis, e, torch.zeros_like(e)).amax(-1, keepdim=True)
        coef = coef + torch.expm1(2 * E)
    return p, p * coef


class Fwd64:
    """attn_fwd64's result.  s, vis: float64 logits and visible keys [H, B, T, T]; mag, ulp: the tau-proportional and
    the fixed part of the logit bound; keep / dscale: dropout; v: [H, B, T, hd] values."""

    def __init__(self, **kw):
        self.__dict__.update(kw)
        self.p64, _ = softmax64(self.s, self.vis)
        self.pd64 = self.p64 * self.keep * self.dscale
        self.ctx64 = self.pd64 @ self.v
        self.pv_mag = self.pd64 @ self.v.abs()

    def logit_err(self, tau):
        return tau * self.mag + self.ulp

    def p_bound(self, tau):
        """Bound of the kernel's bf16 P against p64."""
        _, dp = softmax64(self.s, self.vis, self.logit_err(tau))
        return bf16_out(dp, self.p64)

    def ctx_bound(self, tau, tau_acc):
        """Bound of the kernel's bf16 ctx [H, B, T, hd] against ctx64."""
        bp = self.p_bound(tau)
        bpd = self.keep * self.dscale * (bp + (BF_REL * (self.p64 + bp) if self.dscale != 1.0 else 0))
        return bf16_out(bpd @ self.v.abs() + tau_acc * self.pv_mag, self.ctx64)


def attn_fwd64(qu, qv, k, v, pos, B, T, H, lens, drop_p=0.0, seed=0, pos_hstride=None, key_bounds=None, device_seed=0,
               scale=1.0, round_scores=False):
    """Same arguments as espresso_b200.ops.attn_fused_fwd (tensors on one device) -> Fwd64.
    scale / round_scores state the unfused chain instead: s = bf16(scale * q k^T) (no positions)."""
    dev = qu.device
    quh, kh, vh = heads(qu, B, T, H), heads(k, B, T, H), heads(v, B, T, H)
    hd = quh.shape[-1]
    s = scale * (quh @ kh.transpose(-1, -2))
    mag = abs(scale) * (quh.abs() @ kh.abs().transpose(-1, -2))
    ulp = torch.zeros_like(s)
    if round_scores:
        sr = s.to(BF).to(F64)
        ulp = BF_ULP * sr.abs() + U32 * s.abs()
        s = sr
    if pos is not None:
        if pos_hstride is None:
            pos_hstride = hd if pos.shape[1] == H * hd else 0
        qvh = heads(qv, B, T, H)
        ph = torch.stack([pos[:, h * pos_hstride: h * pos_hstride + hd].to(F64) for h in range(H)])  # [H, 2T-1, hd]
        bd = qvh @ ph[:, None].transpose(-1, -2)
        bdm = qvh.abs() @ ph[:, None].abs().transpose(-1, -2)
        bd = bd.to(BF).to(F64)  # the reference keeps BD in the model dtype
        s = s + _skew(bd, T)
        mag = mag + _skew(bdm, T)
        ulp = ulp + BF_ULP * _skew(bd, T).abs() + U32 * s.abs()
    j = torch.arange(T, device=dev)
    if key_bounds is not None:
        lo, hi = key_bounds
        hidden = (j[None, :] < lo.to(dev).long()[:, None]) | (j[None, :] >= hi.to(dev).long()[:, None])
        sh = (s - HIDDEN).to(BF).to(F64)
        ulp = torch.where(hidden, ulp + U32 * (s.abs() + HIDDEN) + BF_ULP * sh.abs(), ulp)
        s = torch.where(hidden, sh, s)
    klen = torch.full((B,), T, device=dev) if lens is None else lens.to(dev).long().clamp(max=T)
    vis = (j[None, :] < klen[:, None])[None, :, None, :].expand(H, B, T, T)
    ld = r8(T)
    keep = keep_mask(seed, (H, B, T, T), ld, drop_p, dev, device_seed).to(F64) if drop_p > 0 else torch.ones_like(s)
    return Fwd64(s=s, vis=vis, mag=mag, ulp=ulp, keep=keep, dscale=dscale(drop_p) if drop_p > 0 else 1.0, v=vh)


class Bwd64:
    def __init__(self, **kw):
        self.__dict__.update(kw)

    def ds_bound(self, tau):
        """Bound of the kernel's bf16 dS against ds64: the dPd and row-dot reductions, the row-term approximation."""
        err = self.p * (self.keep * self.dscale * tau * self.dpd_mag + tau * self.d_mag + self.row_term_err)
        return bf16_out(err, self.ds64)


def attn_bwd64(dctx, ctx, qu, v, p, pd, B, T, H, drop_p=0.0, seed=0, device_seed=0):
    """Backward of the fused forward from the kernel's saved bf16 P (and its own bf16 ctx for the row term), same
    arguments as ops.attn_fused_bwd.  Returns Bwd64 with dpd64, the exact row term D64 = sum_j P_j g_j (g = the dropout
    backward of dPd), the approximation D_ctx = dctx . ctx the kernel uses, ds64 = P (g - D64), dbd64 (skewed copy),
    dk64 = ds64^T qu and dv64 = Pd^T dctx, all [H, B, ., .] float64."""
    dh, ch, quh, vh = heads(dctx, B, T, H), heads(ctx, B, T, H), heads(qu, B, T, H), heads(v, B, T, H)
    pf = p[..., :T].to(F64)
    pdf = pd[..., :T].to(F64)
    dpd = dh @ vh.transpose(-1, -2)
    dpd_mag = dh.abs() @ vh.abs().transpose(-1, -2)
    ld = p.shape[-1]
    if drop_p > 0:
        keep, sc = keep_mask(seed, (H, B, T, T), ld, drop_p, dpd.device, device_seed).to(F64), dscale(drop_p)
    else:
        keep, sc = torch.ones_like(dpd), 1.0
    g = keep * sc * dpd
    D64 = (pf * g).sum(-1, keepdim=True)
    Dctx = (dh * ch).sum(-1, keepdim=True)
    d_mag = (dh.abs() * ch.abs()).sum(-1, keepdim=True)
    ds64 = pf * (g - D64)
    return Bwd64(p=pf, pd=pdf, keep=keep, dscale=sc, dpd64=dpd, dpd_mag=dpd_mag, D64=D64, Dctx=Dctx, d_mag=d_mag,
                 row_term_err=(Dctx - D64).abs(), ds64=ds64, dk64=ds64.transpose(-1, -2) @ quh,
                 dv64=pdf.transpose(-1, -2) @ dh)


def attn_grad64(qu, qv, k, v, pos, B, T, H, lens, dctx, drop_p=0.0, seed=0, pos_hstride=None, device_seed=0):
    """Float64 autograd of (qu, qv, k, v, pos) -> ctx = dropout(softmax(qu k^T + skew(qv pos^T))) v under the kernels'
    dropout mask, no rounding anywhere.  Returns dict of gradients (qu, qv, k, v, pos) for the cotangent dctx, each in the
    layout of its input ([B*T, d] / [2T-1, E])."""
    dev = qu.device
    d = qu.shape[1]
    hd = d // H
    leaves = {n: t.detach().to(F64).clone().requires_grad_(True)
              for n, t in (("qu", qu), ("qv", qv), ("k", k), ("v", v), ("pos", pos)) if t is not None}
    with torch.enable_grad():
        quh = leaves["qu"].reshape(B, T, H, hd).permute(2, 0, 1, 3)
        s = quh @ leaves["k"].reshape(B, T, H, hd).permute(2, 0, 1, 3).transpose(-1, -2)
        if pos is not None:
            if pos_hstride is None:
                pos_hstride = hd if pos.shape[1] == d else 0
            ph = torch.stack([leaves["pos"][:, h * pos_hstride: h * pos_hstride + hd] for h in range(H)])
            bd = leaves["qv"].reshape(B, T, H, hd).permute(2, 0, 1, 3) @ ph[:, None].transpose(-1, -2)
            s = s + _skew(bd, T)
        j = torch.arange(T, device=dev)
        klen = torch.full((B,), T, device=dev) if lens is None else lens.to(dev).long().clamp(max=T)
        vis = (j[None, :] < klen[:, None])[None, :, None, :]
        # an utterance without keys (lens[b] == 0) attends to nothing: P = 0, as in the kernels
        s = s.masked_fill(~vis, -float("inf")).masked_fill((klen == 0)[None, :, None, None], 0.0)
        pr = torch.softmax(s, -1) * (klen > 0).to(F64)[None, :, None, None]
        if drop_p > 0:
            pr = pr * keep_mask(seed, (H, B, T, T), r8(T), drop_p, dev, device_seed).to(F64) * dscale(drop_p)
        ctx = (pr @ leaves["v"].reshape(B, T, H, hd).permute(2, 0, 1, 3)).permute(1, 2, 0, 3).reshape(B * T, d)
        (ctx * dctx.to(F64)).sum().backward()
    return {n: t.grad for n, t in leaves.items()}


# ---- unfused softmax chain (esp_attn_softmax_fwd / _relaxed_fwd / _bwd) ------------------------------------------------
def _vis_rows(H, B, Tq, Tk, lens, causal, dev):
    j = torch.arange(Tk, device=dev)
    klen = torch.full((B,), Tk, device=dev) if lens is None else lens.to(dev).long().clamp(max=Tk)
    vis = (j[None, :] < klen[:, None])[None, :, None, :].expand(H, B, Tq, Tk)
    if causal:
        vis = vis & (j[None, :] <= torch.arange(Tq, device=dev)[:, None])
    return vis


def softmax_fwd64(scores, Tk, lens, causal=False):
    """scores bf16 [H, B, Tq, ld] over Tk keys -> (p64 [H, B, Tq, Tk], bound of the kernel's bf16 P)."""
    H, B, Tq, _ = scores.shape
    vis = _vis_rows(H, B, Tq, Tk, lens, causal, scores.device)
    p, dp = softmax64(scores[..., :Tk].to(F64), vis)
    return p, bf16_out(dp, p)


def softmax_relaxed_fwd64(scores, Tk, lens, w):
    """(p64, bound of P, r64 = (1 - w) p64 + w / Tk over every padded key, bound of the kernel's relaxed bf16 values)."""
    p, bp = softmax_fwd64(scores, Tk, lens)
    r = (1 - w) * p + w / Tk
    # keep_w * P is rounded to bf16, + add_w, rounded again; w / Tk and 1 - w are fp32 constants
    br = bf16_out((1 - w) * bp + BF_REL * (1 - w) * (p + bp) + U32 * (1 + w / Tk), r)
    return p, bp, r, br


def softmax_bwd64(p, dp_drop, Tk, drop_p=0.0, seed=0, device_seed=0):
    """dS = P (g - sum_j P g) with g the dropout backward of dPd, from the bf16 inputs: (ds64 [H, B, Tq, Tk], bound of
    the kernel's fp32 dS before its bf16 cast per unit tau, i.e. P (|g| + sum_j P |g|))."""
    H, B, Tq, ld = p.shape
    pf, g = p[..., :Tk].to(F64), dp_drop[..., :Tk].to(F64)
    if drop_p > 0:
        g = g * keep_mask(seed, (H, B, Tq, Tk), ld, drop_p, p.device, device_seed).to(F64) * dscale(drop_p)
    ds = pf * (g - (pf * g).sum(-1, keepdim=True))
    mag = pf * (g.abs() + (pf * g.abs()).sum(-1, keepdim=True))
    return ds, mag


# ---- decode attention ---------------------------------------------------------------------------------------------
class Dec64:
    def __init__(self, **kw):
        self.__dict__.update(kw)
        self.p64, _ = softmax64(self.s, self.vis)
        self.ctx64 = torch.einsum("nht,nthc->nhc", self.p64, self.v)
        self.pv_mag = torch.einsum("nht,nthc->nhc", self.p64, self.v.abs())

    def p_bound(self, tau):
        """Bound of the kernel's fp32 probabilities."""
        return softmax64(self.s, self.vis, tau * self.mag)[1] + U32 * self.p64

    def ctx_bound(self, tau, tau_acc):
        bp = bf16_out(self.p_bound(tau), self.p64)
        return bf16_out(torch.einsum("nht,nthc->nhc", bp, self.v.abs()) + tau_acc * self.pv_mag, self.ctx64)


def decode_self_attn64(q, kv_cache, anc, T, H, scale):
    """Hypothesis n at time t reads cache row anc[t, n] of step t.  -> Dec64 (ctx64 [N, H, hd], p64 [N, H, T])."""
    N, d = q.shape
    hd = d // H
    t = torch.arange(T, device=q.device)[:, None]
    kvs = kv_cache[:T].to(F64)[t, anc[:T].long()]  # [T, N, 2d]
    k = kvs[..., :d].reshape(T, N, H, hd).permute(1, 0, 2, 3)  # [N, T, H, hd]
    v = kvs[..., d:].reshape(T, N, H, hd).permute(1, 0, 2, 3)
    qh = q.to(F64).reshape(N, H, hd)
    s = scale * torch.einsum("nhc,nthc->nht", qh, k)
    mag = abs(scale) * torch.einsum("nhc,nthc->nht", qh.abs(), k.abs())
    return Dec64(s=s, mag=mag, vis=torch.ones_like(s, dtype=torch.bool), v=v)


def decode_self_attn_paths64(q, kv_cache, cells, lens, H, scale):
    """Hypothesis n reads its lens[n] keys, key i at flat cell cells[i, n] of the frame-slot cache kv_cache [S, N, 2d]
    (the path tables of esp_decode_update_paths).  A hypothesis without keys has p64 = 0 and ctx64 = 0.  -> Dec64."""
    N, d = q.shape
    hd = d // H
    S = cells.shape[0]
    T = max(int(lens.max()), 1)
    vis = torch.arange(T, device=q.device)[None, :] < lens.to(q.device).long()[:, None]  # [N, T]
    c = torch.where(vis.t(), cells[:T].long(), torch.zeros_like(cells[:T].long()))       # unused entries: any valid cell
    kvs = kv_cache.reshape(S * kv_cache.shape[1], 2 * d).to(F64)[c]                      # [T, N, 2d]
    k = kvs[..., :d].reshape(T, N, H, hd).permute(1, 0, 2, 3)
    v = kvs[..., d:].reshape(T, N, H, hd).permute(1, 0, 2, 3)
    qh = q.to(F64).reshape(N, H, hd)
    s = scale * torch.einsum("nhc,nthc->nht", qh, k)
    mag = abs(scale) * torch.einsum("nhc,nthc->nht", qh.abs(), k.abs())
    return Dec64(s=s, mag=mag, vis=vis[:, None, :].expand(N, H, T), v=v)


def decode_cross_attn64(q, kv, lens, beam, H, scale):
    """Hypothesis n reads sentence n // beam.  -> Dec64 with weights64 [N, Tk] = the head mean of p64, and its
    bound w_bound(tau)."""
    N, d = q.shape
    hd = d // H
    bsz, Tk, _ = kv.shape
    sent = torch.arange(N, device=q.device) // beam
    kvf = kv.to(F64)[sent]
    k, v = kvf[..., :d].reshape(N, Tk, H, hd), kvf[..., d:].reshape(N, Tk, H, hd)
    qh = q.to(F64).reshape(N, H, hd)
    s = scale * torch.einsum("nhc,nthc->nht", qh, k)
    mag = abs(scale) * torch.einsum("nhc,nthc->nht", qh.abs(), k.abs())
    klen = torch.full((N,), Tk, device=q.device) if lens is None else lens.to(q.device).long()[sent].clamp(max=Tk)
    vis = (torch.arange(Tk, device=q.device)[None, :] < klen[:, None])[:, None, :].expand(N, H, Tk)
    r = Dec64(s=s, mag=mag, vis=vis, v=v)
    r.weights64 = r.p64.mean(1)
    r.w_bound = lambda tau: r.p_bound(tau).mean(1) + (H + 2) * U32 * r.weights64
    return r


def tau_reached(ok, hi):
    """Smallest tau in [0, hi] (to 1 %) with ok(tau) True, or float('inf') when ok(hi) is False.  ok is monotone."""
    if ok(0.0):
        return 0.0
    if not ok(hi):
        return float("inf")
    lo = hi * 1e-9
    if ok(lo):
        return lo
    while hi / lo > 1.01:
        mid = float(np.sqrt(lo * hi))
        lo, hi = (lo, mid) if ok(mid) else (mid, hi)
    return hi
