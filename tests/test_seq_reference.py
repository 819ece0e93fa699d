"""CPU checks of the float64 sequence-side statements in oracle/seq64.py (and decode_self_attn_paths64 in
oracle/attn64.py), each against an independent result: float64 torch autograd of the same math, torch.argmax, the fp32
restatements of oracle/ops_ref.py (bit for bit where the statement is exact, within a few fp32 roundings elsewhere), and
the ancestry-table statement decode_self_attn64."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import attn64 as A
from oracle import block64 as K
from oracle import ops_ref as O
from oracle import seq64 as S

F64, F32, BF = torch.float64, torch.float32, torch.bfloat16


def _bf(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g, dtype=F64) * scale).to(BF)


@pytest.fixture(autouse=True)
def _no_device_seed(monkeypatch):
    """The statements take the call's seed alone; ops_ref would add a device seed left by another test."""
    monkeypatch.setattr(O, "_SEED_T", None)


def _ints(shape, seed, hi):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-hi, hi + 1, shape, generator=g)


# -------------------------------------------------------------------------------------------------------- joint
def test_joint_fwd_statement_is_the_fp32_kernel_form():
    B, T, U1, J = 2, 5, 4, 24
    e, d = _bf((B, T, J), 1), _bf((B, U1, J), 2)
    d[0, 1] = -e[0, 2]                                   # exact zero sums
    e[1, 0, :8] = e[1, 0, :8] * 2.0 ** 30                # exponent gaps beyond fp32's 24 bits
    f = S.joint_fwd64(e, d)
    assert (f[0, 2, 1] == 0).all()
    assert torch.equal(f, O.joint_fwd(e, d).to(F64))
    assert torch.equal(f, torch.relu(e.to(F64)[:, :, None] + d.to(F64)[:, None]).to(BF).to(F64))


@pytest.mark.parametrize("exact", [True, False])
def test_joint_bwd_statement_against_autograd(exact):
    B, T, U1, J = 2, 6, 5, 16
    e, d = _bf((B, T, J), 3), _bf((B, U1, J), 4)
    d[1, 2] = -e[1, 3]                                   # F = 0 exactly: no gradient
    df = _ints((B, T, U1, J), 5, 64).to(BF) if exact else _bf((B, T, U1, J), 5)
    dd0 = torch.randn(B, U1, J, generator=torch.Generator().manual_seed(6))
    er, dr = e.to(F64).requires_grad_(True), d.to(F64).requires_grad_(True)
    torch.relu(er[:, :, None] + dr[:, None]).backward(df.to(F64))
    r = S.joint_bwd64(df, S.joint_fwd64(e, d).to(BF), dd0)
    assert torch.equal(r.de, er.grad) and torch.allclose(r.dd, dr.grad + dd0.to(F64), rtol=0, atol=1e-12)
    de32, dd32 = O.joint_bwd(df, O.joint_fwd(e, d))
    if exact:  # every fp32 sum is exact
        assert torch.equal(de32.to(F64), S.rn(r.de)) and torch.equal(dd32.to(F64), r.dd - dd0.to(F64))
    assert K.tau_reached(de32, r.de, r.de_mag, bf16=True) <= U1 * S.U32
    assert K.tau_reached(dd32 + dd0, r.dd, r.dd_mag) <= (T + 1) * S.U32


# -------------------------------------------------------------------------------------------------------- embedding
@pytest.mark.parametrize("pos_kind,scale,drop", [("sin", 8.0, 0.0), ("learned", 512 ** 0.5, 0.0), (None, 1.0, 0.0),
                                                 ("sin", 512 ** 0.5, 0.1)])
def test_embed_fwd_statement_against_ops_ref(pos_kind, scale, drop):
    Vv, d, B, U, pad = 37, 64, 3, 7, 1
    E = _bf((Vv, d), 7)
    tok = torch.randint(0, Vv, (B * U,), generator=torch.Generator().manual_seed(8), dtype=torch.int32)
    tok[[2, 9, 20]] = pad
    pos = None if pos_kind is None else _bf((U + 3, d), 9, 0.5)
    x = S.embed_fwd64(tok, E, pos, U, scale, pad, drop, 11)
    assert torch.equal(x, O.embed_fwd(tok, E, pos, U, scale, pad, drop_p=drop, seed=11).to(F64))
    if pos is not None and drop == 0:  # a pad row carries no positional term
        assert torch.equal(x[2], S.rn(S.f32(E[pad].to(F64) * S.f32(scale))))


@pytest.mark.parametrize("drop", [0.0, 0.1])
def test_embed_bwd_statement_against_autograd(drop):
    Vv, d, R, pad, scale = 29, 16, 60, 1, 2.0
    tok = torch.randint(0, Vv, (R,), generator=torch.Generator().manual_seed(12), dtype=torch.int32)
    tok[::7] = pad
    dx = _bf((R, d), 13)
    dE0 = torch.randn(Vv, d, generator=torch.Generator().manual_seed(14))
    E = torch.zeros(Vv, d, dtype=F64, requires_grad=True)
    y = F.embedding(tok.long(), E, padding_idx=pad) * S.f32(scale)
    if drop > 0:
        keep = S._embed_keep(15, R, d, drop, "cpu")
        y = y * keep * S.f32(S._rng.scale(drop))
    y.backward(dx.to(F64))
    r = S.embed_bwd64(tok, dx, dE0, scale, pad, drop, 15)
    assert torch.allclose(r.dE, E.grad + dE0.to(F64), rtol=0, atol=1e-12)
    assert torch.equal(r.dE[pad], dE0[pad].to(F64))
    got = dE0.clone()
    O.embed_bwd(tok, dx, got, scale, pad, drop_p=drop, seed=15)
    assert K.tau_reached(got, r.dE, r.dE_mag) <= 8 * R * S.U32


# -------------------------------------------------------------------------------------------------------- argmax
def test_argmax_statement_is_torch_argmax():
    nan, inf = float("nan"), float("inf")
    rows = [[1.0, 3.0, 3.0, -1.0, 0.5], [-inf] * 5, [1.0, nan, 7.0, nan, 2.0], [nan] * 5, [2.0, 2.0, 2.0, 2.0, 2.0],
            [-inf, -inf, -3.0, -inf, -3.0], [0.0, -0.0, 0.0, -1.0, nan], [inf, nan, inf, 1, 1]]
    x = torch.tensor(rows, dtype=F32).to(BF)
    wide = torch.cat([x, torch.full((len(rows), 3), nan).to(BF)], 1)  # columns beyond V are ignored
    for t in (x, wide):
        got = S.argmax_rows64(t, 5)
        assert torch.equal(got, t[:, :5].argmax(-1)), got
        assert torch.equal(got, t[:, :5].to(F64).argmax(-1))
    r = _bf((50, 300), 16)
    r[:, 100] = r.max()                                  # ties at 100 and later copies
    r[:, 200] = r.max()
    assert torch.equal(S.argmax_rows64(r, 300), r.argmax(-1))
    assert torch.equal(S.argmax_rows64(r, 300).to(torch.int32), O.argmax_rows(r, 300))
    assert torch.equal(S.argmax_rows64(r[:, :1], 1), torch.zeros(50, dtype=torch.int64))


# -------------------------------------------------------------------------------------------------------- beam merge
def _merge_cases():
    return [dict(), dict(temperature=0.7), dict(lm="bf", lm_weight=0.45), dict(lm="f32", lm_weight=0.3, lm_is_logits=False),
            dict(prev=True, unk_penalty=0.8), dict(force_eos=True), dict(ban_eos=True), dict(eos_factor=1.3), dict(x="lp")]


@pytest.mark.parametrize("kw", _merge_cases(), ids=lambda k: "-".join("%s=%s" % i for i in k.items()) or "plain")
def test_beam_merge_statement_against_float64_log_softmax_and_ops_ref(kw):
    kw = dict(kw)
    N, V = 6, 50
    x = _bf((N, V), 17, 3.0)
    x_is_logits = kw.pop("x", "logits") == "logits"
    if not x_is_logits:
        x = torch.log_softmax(x.float(), -1)
    x[4, 7] = float("nan")
    x[5] = -float("inf")
    lm = kw.pop("lm", None)
    if lm is not None:
        lm = _bf((N, V), 18, 2.0)
        if lm == "f32" or not kw.get("lm_is_logits", True):
            lm = torch.log_softmax(lm.float(), -1)
    prev = torch.randn(N, generator=torch.Generator().manual_seed(19)) if kw.pop("prev", False) else None
    r = S.beam_merge64(x, V, x_is_logits, prev_scores=prev, lm=lm, **kw)
    # float64 restatement through torch.log_softmax
    it = S.f32(1.0 / np.float32(kw.get("temperature", 1.0)))
    lp = torch.log_softmax(x.to(F64) * it, -1) if x_is_logits else x.to(F64)
    if lm is not None:
        lp = lp + S.f32(kw["lm_weight"]) * (torch.log_softmax(lm.to(F64), -1) if kw.get("lm_is_logits", True) else lm.to(F64))
    fin = torch.isfinite(r.out)
    assert (r.out[~fin] == -float("inf")).all() and (r.out[5] == -float("inf")).all()  # an all -inf row stays -inf
    # a NaN logit makes its whole row -inf (the log-sum-exp is NaN); a NaN log-prob only itself
    assert (r.out[4] == -float("inf")).all() if x_is_logits else r.out[4, 7] == -float("inf")
    assert torch.isfinite(lp[fin]).all()
    want = lp.clone()
    want[:, 3] -= S.f32(kw.get("unk_penalty", 0.0))
    if prev is not None:
        want = want + prev.to(F64)[:, None]
    assert float((r.out[fin] - want[fin]).abs().max()) < 1e-12
    assert (r.err[fin] < 1e-4).all() and (r.err[fin] > 0).all() == (x_is_logits or lm is not None)
    ref = torch.empty(N, V)
    O.beam_merge(x, V, x_is_logits, ref, prev_scores=prev, lm=lm, **kw)
    assert torch.equal(torch.isfinite(ref), fin | r.undecided[:, None])
    assert float(((ref.to(F64) - r.out).abs() - r.err)[fin].max()) <= 4 * S.U32 * float(r.out[fin].abs().max())


def test_beam_merge_eos_gate_margin():
    """The eos_factor gate is decided in float64 outside its bound and left open inside it."""
    V, f, eos, pad = 10, 1.5, 2, 1
    x = torch.log_softmax(torch.randn(4, V, generator=torch.Generator().manual_seed(20)), -1)
    others = torch.ones(V, dtype=torch.bool)
    others[[pad, eos]] = False
    mx = x[:, others].max(-1).values.to(F64)
    x[:, eos] = torch.tensor([f * mx[0] + 1e-3, f * mx[1] - 1e-3, f * mx[2], -80.0]).to(F32)
    r = S.beam_merge64(x, V, False, eos_factor=f, pad=pad, eos=eos)
    assert r.undecided.tolist() == [False, False, True, False]
    assert torch.isfinite(r.out[0, eos]) and r.out[0, eos] == x[0, eos] and r.eos_alt[0] == -float("inf")
    assert r.out[1, eos] == -float("inf") and r.eos_alt[1] == x[1, eos]
    assert r.out[3, eos] == -float("inf")
    ref = torch.empty(4, V)
    O.beam_merge(x, V, False, ref, eos_factor=f, pad=pad, eos=eos)
    assert torch.equal(ref[[0, 1, 3]].to(F64), r.out[[0, 1, 3]])


# -------------------------------------------------------------------------------------------------------- paths attention
def test_decode_self_attn_paths_statement_against_ancestry_statement():
    H, hd, N, T = 2, 16, 5, 9
    d = H * hd
    q, cache = _bf((N, d), 21), _bf((T + 2, N, 2 * d), 22)
    anc = torch.randint(0, N, (T + 2, N), generator=torch.Generator().manual_seed(23), dtype=torch.int32)
    cells = (torch.arange(T + 2)[:, None] * N + anc).to(torch.int32)
    a = A.decode_self_attn64(q, cache, anc, T, H, 0.25)
    p = A.decode_self_attn_paths64(q, cache, cells, torch.full((N,), T, dtype=torch.int32), H, 0.25)
    assert torch.equal(a.ctx64, p.ctx64) and torch.equal(a.ctx_bound(1e-6, 1e-6), p.ctx_bound(1e-6, 1e-6))
    lens = torch.tensor([0, 1, 4, T, 2], dtype=torch.int32)
    p = A.decode_self_attn_paths64(q, cache, cells, lens, H, 0.25)
    assert (p.ctx64[0] == 0).all() and (p.ctx_bound(1e-6, 1e-6)[0] == 0).all()
    ref = O.decode_self_attn(q[2:3], cache[:, 2:3].contiguous(), torch.zeros(T + 2, 1, dtype=torch.int32), 4, H, 0.25)
    cells2 = cells.clone()
    cells2[:4, 2] = torch.arange(4) * N + 2               # hypothesis 2 reads its own row's first four slots
    p = A.decode_self_attn_paths64(q, cache, cells2, lens, H, 0.25)
    assert float((p.ctx64[2].reshape(-1) - ref.to(F64).reshape(-1)).abs().max()) <= 2 ** -7 * float(ref.abs().max())
