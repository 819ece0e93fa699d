"""Float64 statements of the sequence-side kernels: the transducer joint (csrc/rnnt.cu joint_fwd / joint_bwd), the token
embedding and its backward (csrc/lsce.cu embed_fwd / embed_bwd), the row argmax of greedy CTC decoding (csrc/lsce.cu
argmax_rows) and the beam-search merge (csrc/beam.cu beam_merge).  Decode attention over path tables lives with the other
attention statements in oracle/attn64.py (decode_self_attn_paths64).

TEST INFRASTRUCTURE ONLY.  Each function has the signature of its espresso_b200.ops wrapper and works from the kernel's
own bf16 / fp32 inputs, widened exactly; dropout masks come from oracle/dropout_rng.py, so they are the kernels' masks bit
for bit.  Nothing is written: every function returns float64 results on the device of its inputs.

Rounding points, and what is exact:
  * joint forward: RN_bf16(max(e + d, 0)).  The fp32 sum of two bf16 values is exact, or lies within 2^-24 of a bf16
    value and so far from a bf16 rounding midpoint; the kernel's output equals the statement bit for bit.
  * joint backward: denc = RN_bf16(fp32 sum over u), ddec += fp32 atomics over t.  Integer-valued dF (|dF| <= 64) makes
    every fp32 partial sum exact in any order, so both outputs equal the statement exactly.
  * embedding forward: RN_bf16(fp32(fp32(RN_bf16(fp32(E * scale))) + pos) [* dropout scale]), every fp32 step stated as a
    float64 operation (exact for these operands) rounded to fp32.  Bit-exact.
  * embedding backward: dE += fp32(dx * fp32(dropout scale * scale)) by fp32 atomics.  The statement sums the unrounded
    products; the bound tau * (|dE0| + sum |term|) covers the product and the atomic roundings.
  * argmax: torch.argmax's order (NaN above every number, first NaN, first of equal maxima).  Exact.
  * beam merge: fp32 log-sum-exp (expf 2 ulp, logf 1 ulp, a 256-thread fp32 sum), x * fp32(1 / temperature), fp32 adds of the
    LM term scaled by fp32(lm_weight), of the unk penalty and of the previous score.  The bound `err` is analytic, with no
    tau: see beam_merge64.
"""
import numpy as np
import torch

from oracle import dropout_rng as _rng
from oracle.block64 import Result, rn

F64, F32, BF = torch.float64, torch.float32, torch.bfloat16
U32 = 2.0 ** -24            # fp32 unit roundoff
EXPF_REL = 2.0 ** -22       # expf: 2 ulp
LOGF_REL = 2.0 ** -23       # logf: 1 ulp


def f32(x):
    """Round a float64 tensor (or a Python float) to fp32, as float64."""
    if torch.is_tensor(x):
        return x.to(F32).to(F64)
    return float(np.float32(x))


# ---- transducer joint -------------------------------------------------------------------------------------------------
def joint_fwd64(enc, dec):
    """enc [B, T, J], dec [B, U1, J] (bf16) -> RN_bf16(relu(enc[:, :, None] + dec[:, None])) [B, T, U1, J] float64."""
    s = enc.to(F64)[:, :, None, :] + dec.to(F64)[:, None, :, :]
    return rn(s.clamp_min(0.0))


def joint_bwd64(df, f, ddec0=None):
    """df, f [B, T, U1, J] (bf16); ddec0 fp32 [B, U1, J] the gradient the C entry point accumulates onto (None: 0).
    -> Result(de, de_mag, dd, dd_mag): de = sum_u g, dd = ddec0 + sum_t g with g = df * (f > 0), and their tau scales
    sum_u |g| and |ddec0| + sum_t |g|."""
    g = df.to(F64) * (f.to(F64) > 0)
    dd0 = torch.zeros_like(g[:, 0]) if ddec0 is None else ddec0.to(F64)
    return Result(de=g.sum(2), de_mag=g.abs().sum(2), dd=dd0 + g.sum(1), dd_mag=dd0.abs() + g.abs().sum(1))


# ---- token embedding --------------------------------------------------------------------------------------------------
def _embed_keep(seed, R, d, p, device):
    return _rng.keep_mask(seed, _rng.row_major_index(R, d), p).to(device)


def embed_fwd64(tokens, E, pos, U, scale, pad_idx, drop_p=0.0, seed=0):
    """Same arguments as ops.embed_fwd -> x [R, d] float64 (bf16 values), the kernel's output bit for bit.
    Row r takes pos[r % U] unless tokens[r] == pad_idx; dropout index r * d + c."""
    t = tokens.long()
    R, d = t.numel(), E.shape[1]
    a = rn(f32(E.to(F64)[t] * f32(scale)))
    if pos is not None:
        p = pos.to(F64)[torch.arange(R, device=t.device) % U]
        a = f32(a + p * (t != pad_idx).to(F64)[:, None])
    if drop_p > 0:
        keep = _embed_keep(seed, R, d, drop_p, E.device)
        a = torch.where(keep, f32(a * _rng.scale(drop_p)), torch.zeros_like(a))
    return rn(a)


def embed_bwd64(tokens, dx, dE_acc, scale, pad_idx, drop_p=0.0, seed=0):
    """Same arguments as ops.embed_bwd (dE_acc is read, not written) -> Result(dE, dE_mag): dE = dE_acc + sum over the
    non-pad rows r of token v of keep * dx[r] * ds, ds = fp32(dropout scale * scale) the kernel's per-term factor, and the
    tau scale |dE_acc| + sum |dx[r] * ds|."""
    t = tokens.long()
    R, d = dx.shape
    ds = f32(_rng.scale(drop_p) * f32(scale)) if drop_p > 0 else f32(scale)
    g = dx.to(F64) * ds
    if drop_p > 0:
        g = torch.where(_embed_keep(seed, R, d, drop_p, dx.device), g, torch.zeros_like(g))
    live = t != pad_idx
    dE = dE_acc.to(F64).clone().index_add_(0, t[live], g[live])
    mag = dE_acc.to(F64).abs().index_add_(0, t[live], g[live].abs())
    return Result(dE=dE, dE_mag=mag)


# ---- greedy argmax ----------------------------------------------------------------------------------------------------
def argmax_rows64(x, V):
    """x [R, ld] -> int64 [R]: per row over the first V columns, the first NaN if the row holds one, else the first
    index of the maximum (an all -inf row gives 0)."""
    a = x[:, :V].to(F64)
    nan = torch.isnan(a)
    first_nan = nan.to(torch.int8).argmax(-1)  # argmax of a 0/1 row: its first 1
    m = torch.where(nan, torch.full_like(a, -np.inf), a).amax(-1, keepdim=True)
    first_max = (a == m).to(torch.int8).argmax(-1)
    return torch.where(nan.any(-1), first_nan, first_max)


# ---- beam merge -------------------------------------------------------------------------------------------------------
def _lse_err(a, ea, V):
    """Float64 log-sum-exp over the last axis of a (values the kernel holds to within ea) and the bound of the kernel's
    fp32 mx + logf(sum expf(a - mx)): the relative error of the sum (each term's argument off by ea + the rounding of
    mx and of the subtraction, expf's 2 ulp, and the fp32 sum: ceil(V / 256) terms per thread of the 256-thread CTA,
    then a block tree at most 16 deep), then logf's ulp and the final add."""
    m = a.amax(-1, keepdim=True)
    ls = torch.log(torch.exp(a - m).sum(-1, keepdim=True))
    lse = m + ls
    p = torch.exp(a - lse)
    delta = ea + U32 * (m.abs() + (a - m).abs()) * (ea > 0) + U32 * (a - m).abs()
    s_rel = 1.01 * (torch.nan_to_num(p * delta).sum(-1, keepdim=True) + EXPF_REL) + (-(-V // 256) + 16) * U32
    return lse, 1.01 * s_rel + LOGF_REL * ls.abs() + U32 * lse.abs()


def beam_merge64(x, V, x_is_logits, out=None, prev_scores=None, temperature=1.0, lm=None, lm_is_logits=True, lm_weight=0.0,
                 pad=1, unk=3, unk_penalty=0.0, eos=2, force_eos=False, eos_factor=None, ban_eos=False):
    """Same arguments as ops.beam_merge (out is ignored) -> Result:
      out        float64 [N, V]: the candidate table with the float64 eos_factor decision (-inf where masked);
      err        [N, V]: bound of |kernel - out| at the finite entries;
      undecided  [N] bool: rows whose eos_factor gate lies within its bound, where the kernel may decide either way;
      eos_alt    [N]: the eos entry had the gate decided the other way;
      gate_margin, gate_err  [N]: lp_eos - f * max_v lp_v and its bound (the gate is decided where |margin| > err).
    The statement scales logits by fp32(1 / temperature), as the kernel does.  err is analytic: U32 of each product, the
    log-sum-exp bound of _lse_err, and U32 of the result of each fp32 add."""
    xv = x[:, :V].to(F64)
    it = float(np.float32(1.0) / np.float32(temperature))
    if x_is_logits:
        a = xv * it
        ea = U32 * a.abs() if it != 1.0 else torch.zeros_like(a)
        lse, e_lse = _lse_err(a, ea, V)
        lp = a - lse
        err = ea + e_lse + U32 * lp.abs()
    else:
        lp, err = xv.clone(), torch.zeros_like(xv)
    if lm is not None:
        lv = lm[:, :V].to(F64)
        if lm_is_logits:
            lse_l, e_lse_l = _lse_err(lv, torch.zeros_like(lv), V)
            t = lv - lse_l
            et = e_lse_l + U32 * t.abs()
        else:
            t, et = lv, torch.zeros_like(lv)
        w = f32(lm_weight)
        lp = lp + w * t
        err = err + abs(w) * et + U32 * (w * t).abs() + U32 * lp.abs()
    ninf = torch.full_like(lp, -np.inf)
    lp = torch.where(torch.isnan(lp), ninf, lp)
    lp[:, pad] = -np.inf
    if unk_penalty != 0.0:
        lp[:, unk] = lp[:, unk] - f32(unk_penalty)
        err[:, unk] = err[:, unk] + U32 * lp[:, unk].abs()
    if force_eos:
        keep_eos = lp[:, eos].clone()
        lp[:] = -np.inf
        lp[:, eos] = keep_eos
    N = lp.shape[0]
    fin = torch.isfinite(lp)
    err = torch.where(fin, err, torch.zeros_like(err))
    undecided = torch.zeros(N, dtype=torch.bool, device=lp.device)
    eos_alt = lp[:, eos].clone()
    gate_margin = gate_err = torch.zeros(N, dtype=F64, device=lp.device)
    if eos_factor is not None and not force_eos:
        f = f32(eos_factor)
        mx = lp.amax(-1)
        e = lp[:, eos]
        fmx = f * mx
        gate_err = err[:, eos] + abs(f) * err.amax(-1) + U32 * torch.nan_to_num(fmx.abs(), posinf=0.0)
        both = torch.isfinite(e) & torch.isfinite(fmx)
        gate_margin = e - fmx
        undecided = both & (gate_margin.abs() <= gate_err)
        drop = e < fmx
        eos_alt = torch.where(drop, e, ninf[:, 0])
        lp[:, eos] = torch.where(drop, ninf[:, 0], e)
    if ban_eos:
        lp[:, eos] = -np.inf
        undecided[:] = False
    if prev_scores is not None:
        pv = prev_scores.to(F64)[:, None]
        lp = lp + pv
        eos_alt = eos_alt + pv[:, 0]
        err = err + U32 * torch.where(torch.isfinite(lp), lp.abs(), torch.zeros_like(lp))
    return Result(out=lp, err=err, undecided=undecided, eos_alt=eos_alt, gate_margin=gate_margin, gate_err=gate_err)
