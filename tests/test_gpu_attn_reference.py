"""The attention kernels against the float64 statements of oracle/attn64.py, per element, on every kernel branch:
the fused forward (csrc/attn_fused.cu, with and without positions), the fused backward and its skew kernel
(csrc/attn_fused_bwd.cu), the unfused softmax chain (csrc/elementwise.cu, every NI instance) and decode attention
(csrc/decode_attn.cu).  Outputs sit between NaN-payload sentinels; every case writes achieved error against its bound
through the `parity` fixture.

Bounds: per-element forms of oracle/attn64.py with the fp32 reduction tau below, each about 2x the largest value reached
on an NVIDIA H100 80GB HBM3 (700 W power limit); a tau that reached 0 (the bf16 roundings bound every element on their own) stays at its
analytic value.  A wrong W half, a skew off by one column, a dropout comparison off by one lane value or a row term of 0
moves some element by far more than one bf16 ulp of its value and fails here."""
import ctypes as C
import types

import pytest
import torch

from oracle import attn64 as A
from oracle import dropout_rng as rng

pytestmark = pytest.mark.gpu

BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
TAU_LOGIT = 4e-6   # fp32 logits per unit of |qu||k| + |qv||pos|: reached 0 (the bf16 terms cover every P), so the
                   # analytic 64 * 2^-24 of a 64-term fp32 dot product
TAU_ACC = 1e-6     # fp32 P V, dK and dV reductions per unit of magnitude: reached 4.5e-7 (P V, T = 1025)
TAU_DS = 1.1e-7    # dS (fused: dPd and row-dot reductions; unfused: the softmax backward's row dot): reached 5.5e-8
TAU_DEC = 8e-6     # decode attention's sequential fp32 dot products: reached 0, analytic 128 * 2^-24 (hd 128)
SM_RATIO = 1.0     # unfused softmax: achieved error / bound (exact bf16 logits: the bound has no tau); reached 0.99
GRAD_REL = 1.25e-2  # composition: ||g - g64|| / ||g64|| of every input gradient; reached 6.1e-3 (bf16 P, dS, outputs)
ROW_TERM = 2.5e-2  # fused backward: max P |dctx . ctx - sum_j P g| / max |dS|; reached 1.0e-2
SENT16 = 0x7FA5    # a NaN payload no kernel produces
SENT32 = 0x7FC0DEAD


@pytest.fixture(scope="module", autouse=True)
def _env():
    from espresso_b200 import ops

    assert torch.cuda.is_available()
    saved = ops._SEED_T
    ops.set_seed_tensor(None)
    yield
    ops.set_seed_tensor(saved)


def _ops():
    from espresso_b200 import ops

    return ops


def _lib():
    from espresso_b200 import lib

    return lib


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(BF)


def _sentinel(n, dtype=BF):
    t = torch.empty(n, device="cuda", dtype=dtype)
    t.view(torch.int16 if dtype == BF else torch.int32).fill_(SENT16 if dtype == BF else SENT32)
    return t


def _boxed(shape, dtype=BF, pad=64):
    """A tensor of `shape` inside a flat sentinel buffer with `pad` sentinels on either side -> (buffer, view)."""
    n = 1
    for s in shape:
        n *= s
    buf = _sentinel(n + 2 * pad, dtype)
    return buf, buf[pad:pad + n].view(shape)


def _untouched(buf, view, what):
    flat = buf.reshape(-1)
    mark = torch.zeros(flat.numel(), dtype=torch.bool, device=buf.device)
    idx = torch.arange(flat.numel(), device=buf.device)
    mark[idx.as_strided(view.shape, view.stride(), view.storage_offset() - buf.storage_offset()).reshape(-1)] = True
    bits = flat.view(torch.int16 if buf.dtype == BF else torch.int32)
    bad = (~mark) & (bits != (SENT16 if buf.dtype == BF else SENT32))
    assert not bad.any(), "%s: %d elements written outside the output" % (what, int(bad.sum()))


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _fwd_raw(qu, qv, k, v, pos, B, T, H, lens, kb, ctx, p, pd, ldp, drop, seed, hstride, hd=64, seed_t=None):
    lo, hi = kb if kb is not None else (None, None)
    return _lib().load().esp_attn_fused_fwd(
        _p(qu), _p(qv), qu.stride(0), _p(k), _p(v), k.stride(0), _p(pos), pos.stride(0) if pos is not None else 0, hstride,
        B, T, H, hd, _p(lens), _p(lo), _p(hi), _p(ctx), H * hd, _p(p), _p(pd), ldp, drop, seed, _p(seed_t), _stream())


def _bwd_raw(dctx, ctx, qu, v, p, pd, B, T, H, drop, seed, ws, ds, dbd, ldbd, dk, dv):
    return _lib().load().esp_attn_fused_bwd(
        _p(dctx), _p(ctx), dctx.stride(0), _p(qu), qu.stride(0), _p(v), v.stride(0), _p(p), _p(pd), p.shape[-1], B, T, H, 64,
        drop, seed, None, _p(ws), _p(ds), _p(dbd), ldbd, _p(dk), _p(dv), dk.stride(0), _stream())


def _rows(x, B, T, H):
    """[B*T, H*hd] -> [H, B, T, hd] float64."""
    return A.heads(x, B, T, H)


def _tau(err, bound_fn, hi):
    return A.tau_reached(lambda t: bool((err <= bound_fn(t)).all()), hi)


def _acc_tau(got, val, mag):
    """Smallest tau with |got - val| <= tau * mag + bf16 rounding of val (bf16 outputs); 0-magnitude elements exact."""
    ex = (got.to(F64) - val).abs() - A.BF_REL * val.abs()
    zero = mag == 0
    assert not (ex[zero] > 0).any(), "non-zero error where the magnitude is 0"
    return float((ex.clamp_min(0) / torch.where(zero, torch.ones_like(mag), mag)).max()) if ex.numel() else 0.0


# ------------------------------------------------------------------------------------------------ inputs
def _lens(kind, B, T):
    if kind == "full":
        return None
    vals = {"ragged": [T - (b * 37) % max(T, 1) for b in range(B)], "one": [1] * B, "128": [128] * B, "129": [129] * B,
            "over": [T + 5 + b for b in range(B)], "mixed0": [T if b % 2 == 0 else 0 for b in range(B)]}[kind]
    return torch.tensor([max(1, x) if kind != "mixed0" else x for x in vals], dtype=torch.int32, device="cuda")


def _key_bounds(kind, T):
    if kind is None:
        return None
    i = torch.arange(T)
    if kind == "chunk":  # chunk streaming: chunk of 16 frames, one chunk of left context, none to the right
        c = i // 16
        lo, hi = (c - 1).clamp_min(0) * 16, ((c + 1) * 16).clamp_max(T)
    else:                # limited context: 12 frames left, 3 right
        lo, hi = (i - 12).clamp_min(0), (i + 4).clamp_max(T)
    return lo.to(torch.int32).cuda(), hi.to(torch.int32).cuda()


def _make(B, T, H, posk, seed):
    """qu, qv [B*T, d]; k, v views into a fused qkv buffer (ldkv = 3d); pos per-head, shared (pos_hstride 0) or none, as
    a column view of a wider table (ldpos > width)."""
    d = H * 64
    qu, qv = _rand((B * T, d), seed, 0.25), _rand((B * T, d), seed + 1, 0.25)
    qkv = _rand((B * T, 3 * d), seed + 2)
    pos = None
    hstride = 0
    if posk != "none":
        w = d if posk == "rel" else 64
        pos = _rand((2 * T - 1, w + 24), seed + 3)[:, 8:8 + w]
        hstride = 64 if posk == "rel" else 0
    return qu, qv, qkv[:, d:2 * d], qkv[:, 2 * d:], pos, hstride


# T sweep x (H, B), lens, positions, key ranges, dropout
FWD = []
for _T in [1, 2, 8, 9, 63, 64, 65, 127, 128, 129, 255, 256, 257, 407, 875, 1024, 1025, 1280]:
    _H, _B = {1: (16, 3), 2: (8, 24), 8: (2, 5), 9: (1, 7)}.get(_T, (2, 2) if _T > 400 else (8, 3))
    FWD.append((_T, _H, _B, "ragged" if _T > 9 else "full", "rel", 0.0, None))
    FWD.append((_T, _H, _B, "full", "none", 0.1, None))
FWD += [
    (2049, 1, 1, "ragged", "none", 0.0, None),
    (129, 2, 3, "one", "rel", 0.1, None),
    (200, 2, 2, "128", "shared", 0.5, None),
    (200, 2, 2, "129", "rel", 0.0, "chunk"),
    (300, 2, 2, "over", "shared", 0.1, "context"),
    (257, 1, 2, "ragged", "none", 0.5, "chunk"),
    (65, 2, 2, "mixed0", "rel", 0.1, None),
    (130, 1, 2, "mixed0", "none", 0.0, None),
]


def _case_id(c):
    return "T%d_H%d_B%d_%s_%s_p%g%s" % (c[0], c[1], c[2], c[3], c[4], c[5], "_" + c[6] if c[6] else "")


def _run_fwd(case, seed, dev_seed=None):
    T, H, B, lk, posk, drop, kbk = case
    d = H * 64
    qu, qv, k, v, pos, hs = _make(B, T, H, posk, seed)
    lens, kb = _lens(lk, B, T), _key_bounds(kbk, T)
    ldp = A.r8(T)
    cbuf, ctx = _boxed((B * T, d))
    pbuf, P = _boxed((H, B, T, ldp))
    pdbuf, Pd = _boxed((H, B, T, ldp))
    seed_t = None
    if dev_seed is not None:
        seed_t = torch.tensor([dev_seed], dtype=torch.int64, device="cuda")
    _lib().check(_fwd_raw(qu, qv if pos is not None else None, k, v, pos, B, T, H, lens, kb, ctx, P, Pd if drop else None,
                          ldp, drop, seed, hs, seed_t=seed_t))
    torch.cuda.synchronize()
    return dict(qu=qu, qv=qv, k=k, v=v, pos=pos, hs=hs, lens=lens, kb=kb, ldp=ldp, cbuf=cbuf, ctx=ctx, pbuf=pbuf, P=P,
                pdbuf=pdbuf, Pd=Pd if drop else P, seed_t=seed_t)


@pytest.mark.parametrize("case", FWD, ids=_case_id)
def test_fused_fwd_vs_float64(case, parity):
    T, H, B, lk, posk, drop, kbk = case
    seed = 1000 + T
    dev_seed = 7 if drop == 0.1 and posk == "rel" else None  # graph-replay form: seed + *seed_ptr
    r_ = _run_fwd(case, seed, dev_seed)
    ctx, P, Pd = r_["ctx"], r_["P"], r_["Pd"]
    _untouched(r_["cbuf"], ctx, "ctx")
    _untouched(r_["pbuf"], P, "P")
    if drop:
        _untouched(r_["pdbuf"], Pd, "Pd")
    ref = A.attn_fwd64(r_["qu"], r_["qv"], r_["k"], r_["v"], r_["pos"], B, T, H, r_["lens"], drop, seed,
                       pos_hstride=r_["hs"], key_bounds=r_["kb"], device_seed=dev_seed or 0)
    name = "fused fwd %s %s" % ("pos" if posk != "none" else "nopos", _case_id(case))
    assert (P[..., T:] == 0).all() and (Pd[..., T:] == 0).all(), "probability tail columns [T, ldp) not zero"
    Pv = P[..., :T].to(F64)
    err = (Pv - ref.p64).abs()
    parity(name + " P (tau reached)", _tau(err, ref.p_bound, 1.0), TAU_LOGIT)
    # rows sum to 1 (0 without a visible key) within the sum of their bounds
    rs = (Pv.sum(-1) - ref.p64.sum(-1)).abs()
    assert (rs <= ref.p_bound(TAU_LOGIT).sum(-1)).all(), "probability row sums"
    # dropout: Pd = bf16(fp32(P) * scale) on the kept set of dropout_rng, 0 elsewhere -- bit for bit
    if drop:
        want = torch.where(ref.keep > 0, (P[..., :T].float() * rng.scale(drop)).to(BF).float(), torch.zeros_like(Pv).float())
        assert torch.equal(Pd[..., :T].float(), want), "dropped probabilities / keep set differ from dropout_rng"
    # P V with the kernel's own Pd (tight), and ctx against the float64 chain
    c = _rows(ctx, B, T, H)
    pdk = Pd[..., :T].to(F64)
    parity(name + " ctx vs Pd V (err / |Pd||V|)", _acc_tau(c, pdk @ ref.v, pdk @ ref.v.abs()), TAU_ACC)
    ratio = float(((c - ref.ctx64).abs() / ref.ctx_bound(TAU_LOGIT, TAU_ACC).clamp_min(1e-300)).max())
    parity(name + " ctx vs ctx64 (err / bound)", ratio, 1.0)
    # without saved probabilities: the same ctx, bit for bit
    ctx2 = torch.empty_like(ctx)
    _lib().check(_fwd_raw(r_["qu"], r_["qv"] if r_["pos"] is not None else None, r_["k"], r_["v"], r_["pos"], B, T, H,
                          r_["lens"], r_["kb"], ctx2, None, None, r_["ldp"], drop, seed, r_["hs"], seed_t=r_["seed_t"]))
    torch.cuda.synchronize()
    assert torch.equal(ctx2, ctx), "save_probs=False changes ctx"
    if lk == "mixed0":  # an empty utterance: P = 0 and ctx = 0, like decode cross-attention
        for b in range(1, B, 2):
            assert not P[:, b].any() and not ctx.view(B, T, -1)[b].any()


# every forward shape; with positions up to the skew kernel's 1024 frames
BWD = [c for c in FWD if c[4] == "none" or c[0] <= 1024]


@pytest.mark.parametrize("case", BWD, ids=_case_id)
def test_fused_bwd_vs_float64(case, parity):
    T, H, B, lk, posk, drop, kbk = case
    seed = 2000 + T
    r_ = _run_fwd(case, seed)
    d = H * 64
    qu, v, P, Pd, ctx = r_["qu"], r_["v"], r_["P"], r_["Pd"], r_["ctx"]
    dctx = _rand((B * T, d), seed + 9)
    ldp = r_["ldp"]
    ldbd = A.r8(2 * T - 1)
    dsbuf, ds = _boxed((H, B, T, ldp))
    dbdbuf, dbd = _boxed((H, B, T, ldbd))
    qbuf, dqkv = _boxed((B * T, 3 * d))
    ws = torch.empty(H * B * T, device="cuda", dtype=F32)
    with_dbd = posk != "none"
    _lib().check(_bwd_raw(dctx, ctx, qu, v, P, Pd, B, T, H, drop, seed, ws, ds, dbd if with_dbd else None, ldbd,
                          dqkv[:, d:2 * d], dqkv[:, 2 * d:]))
    torch.cuda.synchronize()
    _untouched(dsbuf, ds, "dS")
    _untouched(qbuf, dqkv[:, d:], "dqkv (q slice and outside)")
    if with_dbd:
        _untouched(dbdbuf, dbd, "dBD")
        assert torch.equal(dbd, A.unskew(ds[..., :T], T, ldbd)), "dBD is not the skewed copy of dS"
    else:
        _untouched(dbdbuf, dbd[:0], "dBD (not requested)")
    ref = A.attn_bwd64(dctx, ctx, qu, v, P, Pd, B, T, H, drop, seed)
    name = "fused bwd %s %s" % ("dBD" if with_dbd else "nodBD", _case_id(case))
    dsv = ds[..., :T].to(F64)
    assert not ds[..., T:].any(), "dS tail columns"
    parity(name + " dS (tau reached)", _tau((dsv - ref.ds64).abs(), ref.ds_bound, 1.0), TAU_DS)
    big = float(ref.ds64.abs().max())
    if big > 0:
        parity(name + " row-term error max P|D_ctx - D64| / max|dS|", float((ref.p * ref.row_term_err).max()) / big,
               ROW_TERM)
    quh, dh = _rows(qu, B, T, H), _rows(dctx, B, T, H)
    dk, dv = _rows(dqkv[:, d:2 * d], B, T, H), _rows(dqkv[:, 2 * d:], B, T, H)
    parity(name + " dK vs dS^T qu (err / mag)", _acc_tau(dk, dsv.transpose(-1, -2) @ quh,
                                                        dsv.abs().transpose(-1, -2) @ quh.abs()), TAU_ACC)
    parity(name + " dV vs Pd^T dctx (err / mag)", _acc_tau(dv, ref.dv64, ref.pd.transpose(-1, -2) @ dh.abs()), TAU_ACC)
    if r_["lens"] is not None:
        klen = r_["lens"].long().clamp(max=T)
        pad = torch.arange(T, device="cuda")[None, :] >= klen[:, None]  # [B, T] padded keys
        assert not dk[:, pad].any() and not dv[:, pad].any(), "padded keys got dK / dV"


# ------------------------------------------------------------------------------------------------ composition
def _compose(qu, qv, k, v, pos, B, T, H, dctx, lens):
    """The calls of EncoderEngine.mha_fwd / mha_bwd: fused forward, fused (or, past 1024 frames with positions, unfused)
    score-side backward, then the dq_u, dq_v and dpos GEMMs.  Returns the gradients of (qu, qv, k, v, pos)."""
    ops = _ops()
    d, hd = H * 64, 64
    ctx, Pr, Pd = ops.attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens)
    dqkv = torch.empty(B * T, 3 * d, device="cuda", dtype=BF)
    dq = torch.empty(B * T, d, device="cuda", dtype=BF)
    ldp, ldt = A.r8(2 * T - 1), A.r8(T)
    if T <= 1024:
        dS, dBD = ops.attn_fused_bwd(dctx, ctx, qu, v, Pr, Pd, B, T, H, ldp, dqkv[:, d:2 * d], dqkv[:, 2 * d:])
        ops.gemm(dS, k, dq, T, hd, T, ldt, k.stride(0), d, b_kmajor=False, nb1=H, nb2=B, sA=(B * T * ldt, T * ldt),
                 sB=(hd, T * k.stride(0)), sC=(hd, T * d))
    else:
        from espresso_b200.modules.encoder_engine import EncoderEngine

        eng = types.SimpleNamespace(d=d, H=H, hd=hd, _drop=lambda kind: 0.0, _seed=lambda li, op: 0)
        dBD = EncoderEngine._attend_bwd(eng, dctx, (Pr, Pd, 1.0), qu, d, k, v, k.stride(0), dq, d, dqkv[:, d:2 * d],
                                        dqkv[:, 2 * d:], 3 * d, B, T, T, 0, 10, ldp=ldp)
    dqv = torch.empty(B * T, d, device="cuda", dtype=BF)
    ops.gemm(dBD, pos, dqv, B * T, hd, 2 * T - 1, ldp, pos.stride(0), d, b_kmajor=False, nb1=H, nb2=1,
             sA=(B * T * ldp, 0), sB=(hd, 0), sC=(hd, 0))
    dP = torch.zeros(2 * T - 1, d, device="cuda", dtype=F32)
    ops.gemm(dBD, qv, dP, 2 * T - 1, hd, B * T, ldp, d, d, a_kmajor=False, b_kmajor=False, nb1=H, nb2=1,
             sA=(B * T * ldp, 0), sB=(hd, 0), sC=(hd, 0), accumulate=True)
    return dict(qu=dq, qv=dqv, k=dqkv[:, d:2 * d], v=dqkv[:, 2 * d:], pos=dP), (ctx, Pr, Pd)


@pytest.mark.parametrize("T", [25, 250, 407, 875, 1025])
def test_composition_vs_float64_autograd(T, parity):
    H, d = 8, 512
    B = max(1, 3500 // T) if T < 1025 else 3
    qu, qv, k, v, _, _ = _make(B, T, H, "none", 3000 + T)
    pos = _rand((2 * T - 1, d), 3100 + T)
    lens = torch.tensor([T - (b * 7) % T for b in range(B)], dtype=torch.int32, device="cuda")
    dctx = _rand((B * T, d), 3200 + T)
    got, (ctx, Pr, Pd) = _compose(qu, qv, k, v, pos, B, T, H, dctx, lens)
    torch.cuda.synchronize()
    ref = A.attn_grad64(qu, qv, k, v, pos, B, T, H, lens, dctx)
    path = "fused" if T <= 1024 else "unfused softmax bwd"
    for n, g64 in ref.items():
        rel = float((got[n].to(F64) - g64).norm() / g64.norm())
        parity("composition T'=%d (%s) d%s ||err|| / ||g64||" % (T, path, n), rel, GRAD_REL)
    del ref
    if T <= 1024:  # the fused backward's row term dctx . bf16(ctx) against sum_j P g at this shape
        rb = A.attn_bwd64(dctx, ctx, qu, v, Pr, Pd, B, T, H)
        parity("composition T'=%d row-term error max P|D_ctx - D64| / max|dS|" % T,
               float((rb.p * rb.row_term_err).max()) / float(rb.ds64.abs().max()), ROW_TERM)


# ------------------------------------------------------------------------------------------------ unfused chain
SMX = []
for _ld in [256, 264, 512, 520, 768, 776, 1024, 1032, 1280]:
    SMX.append((37, _ld - 3, _ld, False))        # Tq != Tk, ld = ceil8(Tk)
SMX += [(200, 189, 256, False), (257, 257, 264, True), (1, 1, 8, False), (64, 64, 72, True)]


def _softmax_raw(sc, Tk, lens, causal, drop, seed, relax_w=None):
    """esp_attn_softmax_fwd (or _relaxed_fwd) into sentinel-boxed P and Pd -> (pbuf, p, pdbuf, pd)."""
    H, B, Tq, ld = sc.shape
    pbuf, p = _boxed((H, B, Tq, ld))
    pdbuf, pd = _boxed((H, B, Tq, ld))
    L = _lib().load()
    if relax_w is None:
        rc = L.esp_attn_softmax_fwd(_p(sc), H, B, Tq, Tk, ld, _p(lens), int(causal), _p(p), _p(pd), drop, seed, None,
                                    _stream())
    else:
        rc = L.esp_attn_softmax_relaxed_fwd(_p(sc), H, B, Tq, Tk, ld, _p(lens), _p(p), _p(pd), relax_w, drop, seed, None,
                                            _stream())
    _lib().check(rc)
    torch.cuda.synchronize()
    _untouched(pbuf, p, "softmax P")
    _untouched(pdbuf, pd, "softmax Pd")
    return p, pd


@pytest.mark.parametrize("case", SMX, ids=lambda c: "Tq%d_Tk%d_ld%d%s" % (c[0], c[1], c[2], "_causal" if c[3] else ""))
def test_unfused_softmax_chain(case, parity):
    Tq, Tk, ld, causal = case
    H, B = 2, 4
    sc = torch.full((H, B, Tq, ld), float("nan"), device="cuda", dtype=BF)
    sc[..., :Tk] = _rand((H, B, Tq, Tk), Tk + ld, 3.0)
    # ragged, clamped (> Tk) and empty (0) utterances
    lens = torch.tensor([Tk, max(1, Tk // 2), Tk + 9, 0], dtype=torch.int32, device="cuda")
    lens_c = None if causal else lens
    name = "softmax Tq%d Tk%d ld%d" % case[:3] + (" causal" if causal else "")
    drop, seed = 0.1, 4000 + ld
    p, pd = _softmax_raw(sc, Tk, lens_c, causal, drop, seed)
    p64, bp = A.softmax_fwd64(sc, Tk, lens_c, causal)
    assert not p[..., Tk:].any() and not pd[..., Tk:].any(), "columns [Tk, ld) not zero"
    parity(name + " P (err / bound)", float(((p[..., :Tk].to(F64) - p64).abs() / bp.clamp_min(1e-300)).max()), SM_RATIO)
    keep = A.keep_mask(seed, (H, B, Tq, Tk), ld, drop, "cuda")
    want = torch.where(keep, (p[..., :Tk].float() * rng.scale(drop)).to(BF).float(), torch.zeros(1, device="cuda"))
    assert torch.equal(pd[..., :Tk].float(), want), "softmax dropout differs from dropout_rng"
    if not causal:
        assert not p[:, 3].any() and not pd[:, 3].any(), "an utterance without keys must get P = Pd = 0"
        for w in (0.35, 1.0):
            pr, prd = _softmax_raw(sc, Tk, lens, False, drop, seed, relax_w=w)
            _, _, r64, br = A.softmax_relaxed_fwd64(sc, Tk, lens, w)
            assert torch.equal(pr, p), "relaxed P differs from the plain softmax"
            kw, aw = float(torch.tensor(1.0 - w, dtype=F32)), float(torch.tensor(w / Tk, dtype=F32))
            rv = ((p[..., :Tk].float() * kw).to(BF).float() + aw).to(BF).float()
            assert torch.equal(prd[..., :Tk].float(), torch.where(keep, (rv * rng.scale(drop)).to(BF).float(),
                                                                   torch.zeros(1, device="cuda"))), "relaxed Pd"
            # without keys: w / Tk on every padded key, then the dropout
            ev = (torch.tensor([aw], device="cuda").to(BF).float() * rng.scale(drop)).to(BF).float()
            empty = torch.where(keep[:, 3], ev, torch.zeros(1, device="cuda"))
            assert torch.equal(prd[:, 3, :, :Tk].float(), empty), "relaxed Pd of an empty utterance"
            assert not prd[..., Tk:].any()
            parity(name + " relaxed w=%g (err / bound)" % w,
                   float(((rv.to(F64) - r64).abs() / br.clamp_min(1e-300)).max()), SM_RATIO)
    # backward, with the skewed copy when Tq == Tk, on a row stride ldp > 2T - 1
    dpd = torch.full_like(p, float("nan"))
    dpd[..., :Tk] = _rand((H, B, Tq, Tk), Tk + 1)
    want_dbd = Tq == Tk
    ldp = A.r8(2 * Tk - 1) + 16
    dsbuf, ds = _boxed((H, B, Tq, ld))
    dbdbuf, dbd = _boxed((H, B, Tq, ldp))
    _lib().check(_lib().load().esp_attn_softmax_bwd(_p(p), _p(dpd), H, B, Tq, Tk, ld, _p(ds), _p(dbd) if want_dbd else None,
                                                    ldp, drop, seed, None, _stream()))
    torch.cuda.synchronize()
    _untouched(dsbuf, ds, "softmax dS")
    _untouched(dbdbuf, dbd if want_dbd else dbd[:0], "softmax dBD")
    ds64, mag = A.softmax_bwd64(p, dpd, Tk, drop, seed)
    ex = (ds[..., :Tk].to(F64) - ds64).abs() - A.BF_REL * ds64.abs()
    parity(name + " dS (err / P(|g| + sum P|g|))", float((ex.clamp_min(0) / mag.clamp_min(1e-300)).max()), TAU_DS)
    assert not ds[..., Tk:].any()
    if not causal:
        assert not ds[:, 3].any(), "an utterance without keys must get dS = 0"
    if want_dbd:
        assert torch.equal(dbd, A.unskew(ds[..., :Tk], Tk, ldp)), "dBD is not the skewed copy of dS"


@pytest.mark.parametrize("hd", [16, 128])
def test_attend_switchboard_head_dims(hd, parity):
    """EncoderEngine._attend / _attend_bwd (the unfused chain, any head dim) against float64."""
    from espresso_b200.modules.encoder_engine import EncoderEngine

    H, B, T = 4, 4, 150
    d = H * hd
    eng = types.SimpleNamespace(d=d, H=H, hd=hd, scaling=hd ** -0.5, _drop=lambda kind: 0.0, _seed=lambda li, op: 0)
    q = _rand((B * T, d), 5000 + hd, 0.5)
    qkv = _rand((B * T, 3 * d), 5001 + hd)
    k, v = qkv[:, d:2 * d], qkv[:, 2 * d:]
    lens = torch.tensor([T, 101, 37, 0], dtype=torch.int32, device="cuda")  # the last utterance has no keys
    ctx, saved = EncoderEngine._attend(eng, q, d, k, v, 3 * d, B, T, T, lens, False, 0, 10)
    dctx = _rand((B * T, d), 5002 + hd)
    dq = torch.empty(B * T, d, device="cuda", dtype=BF)
    dqkv = torch.empty(B * T, 3 * d, device="cuda", dtype=BF)
    EncoderEngine._attend_bwd(eng, dctx, saved, q, d, k, v, 3 * d, dq, d, dqkv[:, d:2 * d], dqkv[:, 2 * d:], 3 * d, B, T,
                              T, 0, 10)
    torch.cuda.synchronize()
    empty = slice(3 * T, 4 * T)
    assert not ctx[empty].any() and not dq[empty].any() and not dqkv[empty, d:].any(), \
        "an utterance without keys must get ctx = 0, dq = dK = dV = 0"
    # forward: s = bf16(scaling q k^T), as the score GEMM writes it; ctx against the float64 chain
    ref = A.attn_fwd64(q, None, k, v, None, B, T, H, lens, scale=hd ** -0.5, round_scores=True)
    ratio = float(((_rows(ctx, B, T, H) - ref.ctx64).abs() / ref.ctx_bound(TAU_LOGIT, TAU_ACC).clamp_min(1e-300)).max())
    parity("attend hd%d ctx vs ctx64 (err / bound)" % hd, ratio, 1.0)
    qs = (q.float() * hd ** -0.5).to(F64)  # the gradient of q_scaled = s q, exact in float64
    g = A.attn_grad64(qs, None, k, v, None, B, T, H, lens, dctx)
    for n, got, g64 in (("q", dq, g["qu"] * hd ** -0.5), ("k", dqkv[:, d:2 * d], g["k"]), ("v", dqkv[:, 2 * d:], g["v"])):
        parity("attend hd%d d%s ||err|| / ||g64||" % (hd, n), float((got.to(F64) - g64).norm() / g64.norm()), GRAD_REL)


# ------------------------------------------------------------------------------------------------ decode attention
DEC = [(T, hd) for T in (1, 31, 32, 33, 900, 1280) for hd in (64, 96, 128)]


@pytest.mark.parametrize("T,hd", DEC)
def test_decode_self_attn_follows_ancestry(T, hd, parity):
    H, N = 4, 6
    d = H * hd
    q = _rand((N, d), 6000 + T + hd)
    cache = _rand((T + 2, N, 2 * d), 6001 + T + hd)
    g = torch.Generator(device="cuda").manual_seed(T + hd)
    anc = torch.randint(0, N, (T + 2, N), generator=g, device="cuda", dtype=torch.int32)
    obuf, out = _boxed((N, d))
    _lib().check(_lib().load().esp_decode_self_attn(_p(q), _p(cache), _p(anc), N, H, hd, T, C.c_float(hd ** -0.5), _p(out),
                                                    _stream()))
    torch.cuda.synchronize()
    _untouched(obuf, out, "decode self-attention out")
    ref = A.decode_self_attn64(q, cache, anc, T, H, hd ** -0.5)
    got = out.to(F64).reshape(N, H, hd)
    parity("decode self T=%d hd%d ctx (tau reached)" % (T, hd),
           _tau((got - ref.ctx64).abs(), lambda t: ref.ctx_bound(t, t), 1.0), TAU_DEC)


@pytest.mark.parametrize("T,hd", DEC)
def test_decode_cross_attn_and_weights(T, hd, parity):
    beam, bsz = 3, 3
    N = beam * bsz
    for H in ((1, 8, 32) if hd == 64 else (8,)):
        d = H * hd
        q = _rand((N, d), 7000 + T + hd + H)
        kv = _rand((bsz, T, 2 * d), 7001 + T + hd + H)
        lens = torch.tensor([T, max(1, T // 3), T + 11], dtype=torch.int32, device="cuda")
        obuf, out = _boxed((N, d))
        _lib().check(_lib().load().esp_decode_cross_attn(_p(q), _p(kv), _p(lens), N, beam, H, hd, T, C.c_float(0.125),
                                                         _p(out), _stream()))
        wbuf, w = _boxed((N, T), F32)
        obuf2, out2 = _boxed((N, d))
        _lib().check(_lib().load().esp_decode_cross_attn_weights(_p(q), _p(kv), _p(lens), N, beam, H, hd, T,
                                                                 C.c_float(0.125), _p(out2), _p(w), _stream()))
        torch.cuda.synchronize()
        for b, o in ((obuf, out), (obuf2, out2), (wbuf, w)):
            _untouched(b, o, "decode cross-attention outputs")
        assert torch.equal(out, out2), "weights launch changes the context"
        ref = A.decode_cross_attn64(q, kv, lens, beam, H, 0.125)
        name = "decode cross T=%d hd%d H%d" % (T, hd, H)
        got = out.to(F64).reshape(N, H, hd)
        parity(name + " ctx (tau reached)", _tau((got - ref.ctx64).abs(), lambda t: ref.ctx_bound(t, t), 1.0), TAU_DEC)
        parity(name + " weights (tau reached)", _tau((w.to(F64) - ref.weights64).abs(), ref.w_bound, 1.0), TAU_DEC)
        assert not w[beam:2 * beam, max(1, T // 3):].any(), "padded weights not exactly 0"


# ------------------------------------------------------------------------------------------------ refusals
def test_host_refusals():
    lib = _lib()
    ops = _ops()
    B, T, H = 2, 40, 2
    qu, qv, k, v, pos, _ = _make(B, T, H, "rel", 1)
    ctx = _sentinel(B * T * H * 64).view(B * T, -1)
    p = _sentinel(H * B * T * 136).view(H, B, T, 136)
    # head_dim != 64 on the fused path, also with key ranges
    kb = _key_bounds("chunk", T)
    assert _fwd_raw(qu, qv, k, v, pos, B, T, 4, None, kb, ctx, None, None, 48, 0.0, 0, 32, hd=32) != 0
    assert "head_dim 64" in lib.load().esp_last_error().decode()
    # probability rows wider than the key tiles cover
    assert _fwd_raw(qu, qv, k, v, pos, B, T, H, None, None, ctx, p, None, 136, 0.0, 0, 64) != 0
    assert "128 ceil(T/128)" in lib.load().esp_last_error().decode()
    torch.cuda.synchronize()
    _untouched(ctx, ctx[:0], "refused ctx")
    _untouched(p, p[:0], "refused P")
    # relative-position backward above 1024 frames
    T2 = 1032
    qu2, qv2, k2, v2, pos2, _ = _make(1, T2, 1, "rel", 2)
    c2, P2, _ = ops.attn_fused_fwd(qu2, qv2, k2, v2, pos2, 1, T2, 1, None)
    dk = torch.empty(T2, 64, device="cuda", dtype=BF)
    with pytest.raises(lib.EspressoB200Error, match="at most 1024 frames"):
        ops.attn_fused_bwd(c2, c2, qu2, v2, P2, P2, 1, T2, 1, A.r8(2 * T2 - 1), dk, dk)
    # unfused softmax beyond 1280 keys
    with pytest.raises(lib.EspressoB200Error, match="register softmax limit"):
        ops.attn_softmax_fwd(torch.zeros(1, 1, 2, 1288, device="cuda", dtype=BF), 1288, None)
    with pytest.raises(lib.EspressoB200Error, match="register softmax range"):
        ops.attn_softmax_relaxed_fwd(torch.zeros(1, 1, 2, 1288, device="cuda", dtype=BF), 1288, None, 0.5)
    with pytest.raises(lib.EspressoB200Error, match="softmax-bwd shape"):
        z = torch.zeros(1, 1, 2, 1288, device="cuda", dtype=BF)
        ops.attn_softmax_bwd(z, z, 1288, 2584)
