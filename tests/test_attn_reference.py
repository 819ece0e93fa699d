"""Pins oracle/attn64.py, the float64 yardstick of tests/test_gpu_attn_reference.py, against independent statements on
the CPU: explicit per-element loops, float64 autograd and finite differences, and the fp32 oracle (oracle/ops_ref.py)
that the golden fixtures tie to the reference model."""
import numpy as np
import pytest
import torch

from oracle import attn64 as A
from oracle import dropout_rng as rng
from oracle import ops_ref

F64, BF = torch.float64, torch.bfloat16


def _rand(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(BF)


def _inputs(B, T, H, hd, seed, shared_pos=False):
    d = H * hd
    qu, qv = _rand((B * T, d), seed, 0.4), _rand((B * T, d), seed + 1, 0.4)
    qkv = _rand((B * T, 3 * d), seed + 2)
    pos = _rand((2 * T - 1, hd if shared_pos else d), seed + 3)
    return qu, qv, qkv[:, d:2 * d], qkv[:, 2 * d:], pos


def _explicit_fwd(qu, qv, k, v, pos, B, T, H, lens, hstride, lo=None, hi=None, keep=None, sc=1.0):
    """Per-element loops: s_ij = qu_i . k_j + bf16(qv_i . pos_{(T-1)-i+j}) (+ hidden rounding), softmax, P v."""
    hd = qu.shape[1] // H
    P = torch.zeros(H, B, T, T, dtype=F64)
    ctx = torch.zeros(B * T, H * hd, dtype=F64)
    for h in range(H):
        c = slice(h * hd, (h + 1) * hd)
        pc = slice(h * hstride, h * hstride + hd)
        for b in range(B):
            klen = min(int(lens[b]), T) if lens is not None else T
            for i in range(T):
                r = b * T + i
                s = []
                for j in range(klen):
                    a = float(qu[r, c].double() @ k[b * T + j, c].double())
                    if pos is not None:
                        w = float(qv[r, c].double() @ pos[(T - 1) - i + j, pc].double())
                        a += float(torch.tensor(w, dtype=F64).to(BF).double())
                    if lo is not None and (j < lo[i] or j >= hi[i]):
                        a = float(torch.tensor(a - 9984.0, dtype=F64).to(BF).double())
                    s.append(a)
                if not s:
                    continue
                e = np.exp(np.array(s) - max(s))
                P[h, b, i, :klen] = torch.from_numpy(e / e.sum())
                pd = P[h, b, i, :klen] * (keep[h, b, i, :klen] * sc if keep is not None else 1.0)
                ctx[r, c] = pd @ v[b * T: b * T + klen, c].double()
    return P, ctx


def _ctx_rows(x, B, T, H):
    """[H, B, T, hd] -> [B*T, H*hd]."""
    return x.permute(1, 2, 0, 3).reshape(B * T, -1)


@pytest.mark.parametrize("case", ["pos", "shared_pos", "nopos", "bounds_dropout", "ragged"])
def test_fwd64_matches_explicit_loops(case):
    B, T, H, hd = 2, 9, 2, 8
    qu, qv, k, v, pos = _inputs(B, T, H, hd, 7, shared_pos=case == "shared_pos")
    lens = torch.tensor([9, 5], dtype=torch.int32) if case in ("ragged", "bounds_dropout") else None
    kb = None
    if case == "bounds_dropout":
        kb = (torch.tensor([0, 0, 0, 3, 3, 3, 6, 6, 6], dtype=torch.int32),
              torch.tensor([3, 3, 3, 6, 6, 6, 9, 9, 9], dtype=torch.int32))
    if case == "nopos":
        pos = None
    drop = 0.3 if case == "bounds_dropout" else 0.0
    hstride = (0 if case == "shared_pos" else hd)
    r = A.attn_fwd64(qu, qv, k, v, pos, B, T, H, lens, drop, 11, key_bounds=kb)
    keep = A.keep_mask(11, (H, B, T, T), A.r8(T), drop, "cpu").double() if drop else None
    P, ctx = _explicit_fwd(qu, qv, k, v, pos, B, T, H, lens, hstride, *(kb or (None, None)), keep=keep,
                           sc=A.dscale(drop) if drop else 1.0)
    assert torch.allclose(r.p64, P, rtol=0, atol=1e-12)
    assert torch.allclose(_ctx_rows(r.ctx64, B, T, H), ctx, rtol=0, atol=1e-12)
    # the bound vanishes with exact arithmetic only where P is 0 (masked keys)
    assert (r.p_bound(0.0)[~r.vis] == 0).all()


def test_skew_matches_brute_force():
    T = 13
    full = torch.randn(2, 3, T, 2 * T - 1, dtype=F64)
    got = A._skew(full, T)
    ldp = A.r8(2 * T - 1)
    back = A.unskew(got, T, ldp)
    for i in range(T):
        for j in range(T):
            assert got[..., i, j].equal(full[..., i, (T - 1) - i + j])
            assert back[..., i, (T - 1) - i + j].equal(got[..., i, j])
        mask = torch.ones(ldp, dtype=torch.bool)
        mask[(T - 1) - i: (T - 1) - i + T] = False
        assert (back[..., i, mask] == 0).all()


def _fwd_exact(qu, qv, k, v, pos, B, T, H, lens, keep, sc):
    """Float64 forward without any rounding (the function attn_grad64 differentiates)."""
    hd = qu.shape[1] // H
    q = qu.double().reshape(B, T, H, hd).permute(2, 0, 1, 3)
    s = q @ k.double().reshape(B, T, H, hd).permute(2, 0, 1, 3).transpose(-1, -2)
    if pos is not None:
        ph = pos.double().reshape(2 * T - 1, H, hd).permute(1, 0, 2)
        s = s + A._skew(qv.double().reshape(B, T, H, hd).permute(2, 0, 1, 3) @ ph[:, None].transpose(-1, -2), T)
    if lens is not None:
        s = s.masked_fill((torch.arange(T)[None, :] >= lens.long()[:, None])[None, :, None, :], -float("inf"))
    p = torch.softmax(s, -1) * keep * sc
    return _ctx_rows(p @ v.double().reshape(B, T, H, hd).permute(2, 0, 1, 3), B, T, H)


@pytest.mark.parametrize("drop", [0.0, 0.25])
def test_grad64_matches_finite_differences(drop):
    B, T, H, hd = 2, 6, 2, 4
    qu, qv, k, v, pos = _inputs(B, T, H, hd, 21)
    lens = torch.tensor([6, 4], dtype=torch.int32)
    dctx = torch.randn(B * T, H * hd, dtype=F64)
    g = A.attn_grad64(qu, qv, k, v, pos, B, T, H, lens, dctx, drop, 5)
    keep = A.keep_mask(5, (H, B, T, T), A.r8(T), drop, "cpu").double() if drop else torch.ones(H, B, T, T, dtype=F64)
    sc = A.dscale(drop) if drop else 1.0
    args = dict(qu=qu.double(), qv=qv.double(), k=k.double(), v=v.double(), pos=pos.double())
    h = 1e-6
    for name in args:
        u = torch.randn_like(args[name])
        plus = dict(args, **{name: args[name] + h * u})
        minus = dict(args, **{name: args[name] - h * u})
        fd = ((_fwd_exact(**plus, B=B, T=T, H=H, lens=lens, keep=keep, sc=sc)
               - _fwd_exact(**minus, B=B, T=T, H=H, lens=lens, keep=keep, sc=sc)) * dctx).sum() / (2 * h)
        assert abs(float(fd) - float((g[name] * u).sum())) < 1e-7 * max(1.0, abs(float(fd))), name


def test_grad64_empty_utterance_contributes_nothing():
    """lens[b] == 0: utterance b attends to nothing (P = 0, ctx = 0, as the kernels define it), so its q, k and v get zero
    gradient and every other gradient equals the run without it."""
    B, T, H, hd = 2, 6, 2, 4
    qu, qv, k, v, pos = _inputs(B, T, H, hd, 23)
    dctx = torch.randn(B * T, H * hd, dtype=F64)
    g = A.attn_grad64(qu, qv, k, v, pos, B, T, H, torch.tensor([5, 0], dtype=torch.int32), dctx)
    g1 = A.attn_grad64(qu[:T], qv[:T], k[:T], v[:T], pos, 1, T, H, torch.tensor([5], dtype=torch.int32), dctx[:T])
    for name in ("qu", "qv", "k", "v"):
        assert torch.isfinite(g[name]).all() and (g[name][T:] == 0).all(), name
        assert torch.allclose(g[name][:T], g1[name], rtol=0, atol=1e-13), name
    assert torch.allclose(g["pos"], g1["pos"], rtol=0, atol=1e-13)
    r = A.attn_fwd64(qu, qv, k, v, pos, B, T, H, torch.tensor([5, 0], dtype=torch.int32))
    assert (r.p64[:, 1] == 0).all() and (r.ctx64[:, 1] == 0).all() and (r.ctx_bound(1e-5, 1e-5)[:, 1] == 0).all()


@pytest.mark.parametrize("drop", [0.0, 0.2])
def test_bwd64_matches_autograd(drop):
    """With float64 P, Pd and ctx, attn_bwd64 is the exact backward: dS, dK, dV equal autograd, and the row term the
    kernel uses (dctx . ctx) equals sum_j P_j g_j."""
    B, T, H, hd = 2, 7, 2, 8
    qu, _, k, v, _ = _inputs(B, T, H, hd, 31)
    lens = torch.tensor([7, 3], dtype=torch.int32)
    ld = A.r8(T)
    keep = A.keep_mask(9, (H, B, T, T), ld, drop, "cpu").double() if drop else torch.ones(H, B, T, T, dtype=F64)
    sc = A.dscale(drop) if drop else 1.0
    kk = k.double().requires_grad_(True)
    vv = v.double().requires_grad_(True)
    s = (qu.double().reshape(B, T, H, hd).permute(2, 0, 1, 3) @ kk.reshape(B, T, H, hd).permute(2, 0, 1, 3).transpose(-1, -2))
    s.retain_grad()
    sm = s.masked_fill((torch.arange(T)[None, :] >= lens.long()[:, None])[None, :, None, :], -float("inf"))
    p = torch.softmax(sm, -1)
    ctx = _ctx_rows(p * keep * sc @ vv.reshape(B, T, H, hd).permute(2, 0, 1, 3), B, T, H)
    dctx = torch.randn_like(ctx)
    (ctx * dctx).sum().backward()
    P = torch.zeros(H, B, T, ld, dtype=F64)
    P[..., :T] = p.detach()
    Pd = P.clone()
    Pd[..., :T] = P[..., :T] * keep * sc
    r = A.attn_bwd64(dctx, ctx.detach(), qu, v, P, Pd, B, T, H, drop, 9)
    assert torch.allclose(r.ds64, s.grad, rtol=0, atol=1e-12)
    assert torch.allclose(_ctx_rows(r.dk64, B, T, H), kk.grad, rtol=0, atol=1e-12)
    assert torch.allclose(_ctx_rows(r.dv64, B, T, H), vv.grad, rtol=0, atol=1e-12)
    assert float(r.row_term_err.max()) < 1e-12


@pytest.mark.parametrize("case", ["per_head", "shared", "bounds", "dropout_ragged"])
def test_ops_ref_within_fp32_bounds(case):
    """The fp32 oracle (tied to the reference by the golden fixtures) stays inside attn64's bounds at fp32-level tau."""
    B, T, H, hd = 2, 20, 2, 16
    qu, qv, k, v, pos = _inputs(B, T, H, hd, 41, shared_pos=case == "shared")
    lens = torch.tensor([20, 13], dtype=torch.int32) if case == "dropout_ragged" else None
    kb = None
    if case == "bounds":
        lo = torch.tensor([max(0, i - 4) for i in range(T)], dtype=torch.int32)
        kb = (lo, torch.tensor([min(T, i + 2) for i in range(T)], dtype=torch.int32))
    drop = 0.1 if case == "dropout_ragged" else 0.0
    ctx, p, pd = ops_ref.attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens, drop, 3, key_bounds=kb,
                                        pos_hstride=0 if case == "shared" else None)
    r = A.attn_fwd64(qu, qv, k, v, pos, B, T, H, lens, drop, 3, key_bounds=kb)
    tau = 1e-5
    assert ((p[..., :T].double() - r.p64).abs() <= r.p_bound(tau)).all()
    assert (p[..., T:] == 0).all()
    got = ctx.double().reshape(B, T, H, hd).permute(2, 0, 1, 3)
    assert ((got - r.ctx64).abs() <= r.ctx_bound(tau, tau)).all()
    if drop:
        assert torch.equal(pd[..., :T] != 0, (r.keep > 0) & (p[..., :T] != 0))


def test_softmax_refs_match_torch():
    H, B, Tq, Tk, ld = 2, 2, 5, 11, 24
    sc = _rand((H, B, Tq, ld), 51, 2.0)
    lens = torch.tensor([11, 0], dtype=torch.int32)
    p, bp = A.softmax_fwd64(sc, Tk, lens)
    want = torch.softmax(sc[..., :Tk].double(), -1)
    assert torch.allclose(p[:, 0], want[:, 0], rtol=0, atol=1e-15)
    assert (p[:, 1] == 0).all() and (bp[:, 1] == 0).all()  # no visible key: exactly 0
    sq = _rand((H, B, Tk, ld), 52, 2.0)
    pc, _ = A.softmax_fwd64(sq, Tk, None, causal=True)
    fut = torch.arange(Tk)[None, :] > torch.arange(Tk)[:, None]
    assert torch.allclose(pc, torch.softmax(sq[..., :Tk].double().masked_fill(fut, -float("inf")), -1), rtol=0, atol=1e-15)
    _, _, r, _ = A.softmax_relaxed_fwd64(sc, Tk, lens, 0.35)
    assert torch.allclose(r[:, 0], 0.65 * want[:, 0] + 0.35 / Tk, rtol=0, atol=1e-15)
    assert torch.allclose(r[:, 1], torch.full_like(r[:, 1], 0.35 / Tk), rtol=0, atol=1e-15)
    # backward: dS = P (g - sum P g) equals autograd of the softmax (no dropout)
    s = sc[:, :1, :, :Tk].double().requires_grad_(True)
    g = torch.randn(H, 1, Tq, Tk, dtype=F64)
    (torch.softmax(s, -1) * g).sum().backward()
    P = torch.zeros(H, 1, Tq, ld, dtype=F64)
    P[..., :Tk] = torch.softmax(s.detach(), -1)
    G = torch.zeros_like(P)
    G[..., :Tk] = g
    ds, _ = A.softmax_bwd64(P, G, Tk)
    assert torch.allclose(ds, s.grad, rtol=0, atol=1e-13)


def test_decode_refs_follow_ancestry():
    N, H, hd, Tmax, T, beam = 6, 2, 8, 9, 7, 3
    d = H * hd
    g = torch.Generator().manual_seed(61)
    q = _rand((N, d), 62)
    cache = _rand((Tmax, N, 2 * d), 63)
    anc = torch.randint(0, N, (Tmax, N), generator=g, dtype=torch.int32)
    r = A.decode_self_attn64(q, cache, anc, T, H, 0.3)
    for n in range(N):
        for h in range(H):
            c = slice(h * hd, (h + 1) * hd)
            ks = torch.stack([cache[t, anc[t, n], c].double() for t in range(T)])
            vs = torch.stack([cache[t, anc[t, n], d + h * hd: d + (h + 1) * hd].double() for t in range(T)])
            p = torch.softmax(0.3 * ks @ q[n, c].double(), 0)
            assert torch.allclose(r.p64[n, h], p, rtol=0, atol=1e-14)
            assert torch.allclose(r.ctx64[n, h], p @ vs, rtol=0, atol=1e-13)
    # fp32 oracle within the bounds at fp32-level tau
    got = ops_ref.decode_self_attn(q, cache, anc, T, H, 0.3).double().reshape(N, H, hd)
    assert ((got - r.ctx64).abs() <= r.ctx_bound(1e-5, 1e-5)).all()
    kv = _rand((N // beam, 10, 2 * d), 64)
    lens = torch.tensor([10, 0], dtype=torch.int32)
    rc = A.decode_cross_attn64(q, kv, lens, beam, H, 0.3)
    for n in range(beam):  # sentence 0, every key
        for h in range(H):
            p = torch.softmax(0.3 * kv[0, :, h * hd:(h + 1) * hd].double() @ q[n, h * hd:(h + 1) * hd].double(), 0)
            assert torch.allclose(rc.p64[n, h], p, rtol=0, atol=1e-14)
    assert (rc.p64[beam:] == 0).all() and (rc.ctx64[beam:] == 0).all() and (rc.weights64[beam:] == 0).all()
    assert torch.allclose(rc.weights64[:beam].sum(-1), torch.ones(beam, dtype=F64), rtol=0, atol=1e-14)


def test_tau_reached_bisects():
    assert A.tau_reached(lambda t: t >= 3e-6, 1e-3) == pytest.approx(3e-6, rel=0.02)
    assert A.tau_reached(lambda t: True, 1e-3) == 0.0
    assert A.tau_reached(lambda t: False, 1e-3) == float("inf")
    assert rng.thresh(0.5) == 32768
