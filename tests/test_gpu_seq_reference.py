"""The sequence-side kernels against the float64 statements of oracle/seq64.py and oracle/attn64.py, per element: the
transducer joint forward and backward (csrc/rnnt.cu), the token embedding and its backward, the greedy row argmax
(csrc/lsce.cu), the beam-search merge (csrc/beam.cu) and decode self-attention over path tables (csrc/decode_attn.cu),
then the whole joint network (_JointFn) against float64 autograd.  Outputs sit between NaN-payload sentinels; every
case writes its achieved error against its bound through the `parity` fixture.

Exact cases compare values (+0 equals -0): the joint forward, the embedding forward (with and without dropout), argmax,
and the joint and embedding backward fed integer-valued gradients.  The other bounds are per-element forms with an fp32
reduction tau, each about 2x the largest value reached on an NVIDIA H100 80GB HBM3 (700 W power limit); the beam merge's
bound is analytic (no tau) and its reached fraction is recorded."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import attn64 as A
from oracle import block64 as K
from oracle import seq64 as S
from test_gpu_attn_reference import TAU_DEC

pytestmark = pytest.mark.gpu

BF, F32, F64, I32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
TAU_JOINT = 2e-7      # joint backward, per unit of sum |g|: ddec (T atomics) reached 8.5e-8; denc (U1-term sums) 0,
                      # its bf16 rounding covers every element
TAU_EMB = 5e-7        # embedding backward, per unit of |dE0| + sum |term| (fp32 products and atomics): reached 2.3e-7
BEAM_RATIO = 1.0      # beam merge: achieved error / analytic bound (a rigorous bound): reached 1 - 2^-24 (one fp32
                      # add rounded at a midpoint), 0.31 wherever a log-sum-exp is involved
GRAD_REL = 7.5e-3     # _JointFn composition: ||x - x64|| / ||x64|| of the logits and every gradient: reached 3.8e-3
SENT16 = 0x7FA5       # a NaN payload no kernel produces
SENT32 = 0x7FC0DEAD


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


def _rand(shape, seed, scale=1.0, dtype=BF):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def _ints(shape, seed, hi, dtype=BF):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-hi, hi + 1, shape, generator=g, device="cuda").to(dtype)


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


def _p(t, off=0):
    return None if t is None else C.c_void_p(t.data_ptr() + off)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc):
    _lib().check(rc)
    torch.cuda.synchronize()


def _exact(got, want):
    """Largest |got - want| (0 when equal as values, so +0 == -0); NaN anywhere counts as infinite."""
    d = (got.to(F64) - want.to(F64)).abs()
    return float("inf") if torch.isnan(d).any() else (float(d.max()) if d.numel() else 0.0)


# ------------------------------------------------------------------------------------------------ joint forward
JF = [(2, 7, 5, J) for J in (8, 264, 512, 640, 2056)] + [(4, 875, 101, 512)]


@pytest.mark.parametrize("B,T,U1,J", JF)
def test_joint_fwd_bit_exact(B, T, U1, J, parity):
    e, d = _rand((B, T, J), 100 + J), _rand((B, U1, J), 101 + J)
    d[0, 1] = -e[0, 3]                   # sums exactly 0
    d[B - 1, U1 - 1, : J // 2] = -e[B - 1, 0, : J // 2]
    buf, out = _boxed((B, T, U1, J))
    _check(_lib().load().esp_joint_fwd(_p(e), _p(d), B, T, U1, J, _p(out), _stream()))
    _untouched(buf, out, "joint fwd")
    ref = S.joint_fwd64(e, d)
    assert (ref[0, 3, 1] == 0).all()
    parity("joint fwd B%d T%d U1=%d J%d max |F - F64|" % (B, T, U1, J), _exact(out, ref), 0.0)


# ------------------------------------------------------------------------------------------------ joint backward
# threads per CTA: J/8 rounded up to a warp below 256 (J 8: 1 of 32 lanes, 200: 25, 264: 33 -> 64), else 256 in a loop
JB = [(1, 1, 1, 8), (2, 1, 256, 200), (2, 3, 600, 264), (3, 5, 7, 2056), (2, 9, 256, 512), (4, 875, 101, 512)]


@pytest.mark.parametrize("exact", [True, False], ids=["int", "rand"])
@pytest.mark.parametrize("B,T,U1,J", JB)
def test_joint_bwd(B, T, U1, J, exact, parity):
    e, d = _rand((B, T, J), 200 + J), _rand((B, U1, J), 201 + J)
    d[0, 0] = -e[0, 0]                   # F = 0 exactly: masked
    f = S.joint_fwd64(e, d).to(BF)
    df = _ints((B, T, U1, J), 202 + J, 64) if exact else _rand((B, T, U1, J), 202 + J)
    dd0 = _ints((B, U1, J), 203 + J, 1000, F32) if exact else _rand((B, U1, J), 203 + J, 1.0, F32)
    bde, de = _boxed((B, T, J))
    bdd, dd = _boxed((B, U1, J), F32)
    dd.copy_(dd0)                        # the C entry point accumulates into ddec
    _check(_lib().load().esp_joint_bwd(_p(df), _p(f), B, T, U1, J, _p(de), _p(dd), _stream()))
    _untouched(bde, de, "joint bwd denc")
    _untouched(bdd, dd, "joint bwd ddec")
    r = S.joint_bwd64(df, f, dd0)
    name = "joint bwd B%d T%d U1=%d J%d" % (B, T, U1, J)
    if exact:
        parity(name + " int dF: max |denc - RN(denc64)|", _exact(de, S.rn(r.de)), 0.0)
        parity(name + " int dF: max |ddec - ddec64|", _exact(dd, r.dd), 0.0)
    else:
        parity(name + " denc (tau reached)", K.tau_reached(de, r.de, r.de_mag, bf16=True), TAU_JOINT)
        parity(name + " ddec (tau reached)", K.tau_reached(dd, r.dd, r.dd_mag), TAU_JOINT)


# ------------------------------------------------------------------------------------------------ embedding forward
def _sinusoidal(n, d, pad):
    """fairseq's SinusoidalPositionalEmbedding table (row `pad` zero) as bf16."""
    half = d // 2
    f = torch.exp(torch.arange(half, dtype=F64) * -(np.log(10000.0) / (half - 1)))
    a = torch.arange(n, dtype=F64)[:, None] * f[None, :]
    t = torch.cat([torch.sin(a), torch.cos(a)], 1)
    t[pad] = 0
    return t.to(BF).cuda()


EF = [(d, pk, sc, p) for d in (8, 64, 512, 1024) for pk in ("sin", "learned", None) for sc, p in (("sqrt", 0.0), ("one", 0.1))]
EF += [(512, "sin", "sqrt", 0.0, "step"), (64, "learned", "one", 0.1, "step"), (512, "sin", "sqrt", 0.1, "big"),
       (64, "sin", "one", 0.0, "wrap")]


@pytest.mark.parametrize("case", EF, ids=lambda c: "-".join(str(x) for x in c))
def test_embed_fwd_bit_exact(case, parity):
    d, pk, sc, p = case[:4]
    form = case[4] if len(case) > 4 else "rows"
    Vv, pad = 1000, 1
    # rows: B = 3 sentences of U = 37; step: one decode step (U = N, positions gathered per row); big: 24 x 875 rows
    # (the grid-stride loop runs several times); wrap: R = 50 rows over U = 7 (r % U wraps mid-sentence)
    R, U = {"rows": (111, 37), "step": (12, 12), "big": (21000, 875), "wrap": (50, 7)}[form]
    E = _rand((Vv, d), 300 + d)
    tok = torch.randint(0, Vv, (R,), generator=torch.Generator(device="cuda").manual_seed(301), device="cuda",
                        dtype=I32)
    tok[::5] = pad
    scale = float(np.sqrt(d)) if sc == "sqrt" else 1.0
    if pk is None:
        pos = None
    else:
        table = _sinusoidal(1024 + 2, d, pad) if pk == "sin" else _rand((1024, d), 302 + d)
        if form == "step":  # each hypothesis at its own position
            pos = table[torch.randint(2, 1000, (U,), generator=torch.Generator(device="cuda").manual_seed(303),
                                      device="cuda")].contiguous()
        else:
            pos = table[2:2 + U].contiguous()
    buf, x = _boxed((R, d))
    _check(_lib().load().esp_embed_fwd(_p(tok), _p(E), _p(pos), U, d, scale, R, pad, _p(x), p, 77, None, _stream()))
    _untouched(buf, x, "embed fwd")
    ref = S.embed_fwd64(tok, E, pos, U, scale, pad, p, 77)
    parity("embed fwd d%d pos=%s scale=%s p=%.1f %s max |x - x64|" % (d, pk, sc, p, form), _exact(x, ref), 0.0)


# ------------------------------------------------------------------------------------------------ embedding backward
def _zipf_tokens(R, Vv, seed):
    """Tokens with P(k) ~ (k + 1)^-1.5: token 0 fills about 38 % of the rows, token 1 (the pad) about 13 %."""
    w = (torch.arange(Vv, dtype=F64) + 1) ** -1.5
    g = torch.Generator().manual_seed(seed)
    return torch.multinomial(w, R, replacement=True, generator=g).to(I32).cuda()


@pytest.mark.parametrize("kind", ["int", "rand", "rand-drop"])
def test_embed_bwd(kind, parity):
    Vv, d, R, pad = 1000, 512, 40000, 1
    tok = _zipf_tokens(R, Vv, 400)
    assert int((tok == 0).sum()) > 10 ** 4
    if kind == "int":  # a power-of-two scale: every product and every fp32 partial sum is exact
        scale, p = 0.5, 0.0
        dx, dE0 = _ints((R, d), 401, 64), _ints((Vv, d), 402, 1000, F32)
    else:
        scale, p = float(np.sqrt(d)), (0.1 if kind == "rand-drop" else 0.0)
        dx, dE0 = _rand((R, d), 401), _rand((Vv, d), 402, 3.0, F32)
    buf, dE = _boxed((Vv, d), F32)
    dE.copy_(dE0)
    _check(_lib().load().esp_embed_bwd(_p(tok), _p(dx), d, scale, R, pad, _p(dE), p, 88, None, _stream()))
    _untouched(buf, dE, "embed bwd")
    r = S.embed_bwd64(tok, dx, dE0, scale, pad, p, 88)
    assert torch.equal(dE[pad], dE0[pad]), "the pad row received a gradient"
    name = "embed bwd %s R%d d%d" % (kind, R, d)
    if kind == "int":
        parity(name + " max |dE - dE64|", _exact(dE, r.dE), 0.0)
    else:
        parity(name + " (tau reached)", K.tau_reached(dE, r.dE, r.dE_mag), TAU_EMB)


# ------------------------------------------------------------------------------------------------ argmax
def _argmax_rows(V, R, seed):
    """R rows over V columns: random, exact ties, all -inf, one NaN, several NaN, all NaN, -inf ties with a finite max."""
    x = _rand((R, V), seed, 3.0, F32)
    nan, inf = float("nan"), float("inf")
    g = torch.Generator().manual_seed(seed)
    for r in range(R):
        kind = r % 8
        cols = torch.randint(0, V, (4,), generator=g).tolist()
        if kind == 1:
            x[r, cols] = x[r].max() + 1.0                  # exact ties, first one wins
        elif kind == 2:
            x[r] = -inf
        elif kind == 3:
            x[r, cols[0]] = nan
        elif kind == 4:
            x[r, cols] = nan
        elif kind == 5:
            x[r] = nan
        elif kind == 6:
            x[r] = -inf
            x[r, cols[1:]] = 2.0
        elif kind == 7:
            x[r] = 5.0                                     # all equal
    return x.to(BF)


@pytest.mark.parametrize("V,R", [(1, 16), (127, 64), (128, 64), (129, 64), (5004, 64), (32000, 32), (5004, 24 * 875)])
def test_argmax_rows_exact(V, R, parity):
    ld = A.r8(V) + 8
    x = torch.full((R, ld), float("nan"), device="cuda", dtype=BF)  # NaN beyond column V must be ignored
    x[:, :V] = _argmax_rows(V, R, 500 + V)
    buf, out = _boxed((R,), I32)
    _check(_lib().load().esp_argmax_rows(_p(x), ld, V, R, _p(out), _stream()))
    _untouched(buf, out, "argmax out")
    ref = S.argmax_rows64(x, V)
    assert int(out.min()) >= 0 and int(out.max()) < V, "index outside [0, V): %d" % int(out.max())
    parity("argmax V%d R%d rows differing" % (V, R), int((out.long() != ref).sum()), 0)


def test_ctc_greedy_decoder_on_nan_rows():
    """A diverged model's NaN frames decode to in-range tokens, as torch.argmax decides them."""
    from test_host_orchestration import _Task
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    B, T, V = 3, 40, 50
    out = _rand((B, T, 56), 600, 3.0)
    out[0] = float("nan")                                  # all NaN
    out[1, 5:9, 7] = float("nan")                          # a NaN in some frames
    dec = CTCDecoder(_Task(V).target_dictionary)
    toks, _, _ = dec._greedy(out, V, [T, T, 20])
    am = S.argmax_rows64(out.reshape(B * T, 56), V).view(B, T).cpu()
    assert int(toks.min()) >= 0 and int(toks.max()) < V
    for b, n in enumerate([T, T, 20]):
        seq = torch.unique_consecutive(am[b, :n])
        seq = seq[seq != dec.blank]
        assert toks[b][: seq.numel()].tolist() == seq.tolist()
        assert (toks[b][seq.numel():] == dec.pad).all()


# ------------------------------------------------------------------------------------------------ beam merge
BM = [dict(V=50), dict(V=50, temperature=0.7), dict(V=50, x="f32"), dict(V=50, x="lp"), dict(V=3),
      dict(V=5004, lm="bf", lm_weight=0.45), dict(V=5004, lm="f32", lm_weight=0.3),
      dict(V=5004, lm="lp", lm_weight=0.5, lm_is_logits=False), dict(V=5004, prev=True, unk_penalty=0.8),
      dict(V=10000, force_eos=True, prev=True), dict(V=10000, ban_eos=True), dict(V=10000, eos_factor=1.3),
      dict(V=32000, temperature=1.3, lm="bf", lm_weight=0.2, prev=True, eos_factor=2.0), dict(V=32000, x="lp", prev=True)]


def _merge_inputs(c, N, seed):
    c = dict(c)
    V = c.pop("V")
    ld = A.r8(V) + 8
    kind = c.pop("x", "bf")
    x = torch.full((N, ld), float("nan"), device="cuda", dtype=F32 if kind != "bf" else BF)
    v = _rand((N, V), seed, 3.0, F32)
    x[:, :V] = torch.log_softmax(v, -1) if kind == "lp" else v.to(x.dtype)
    x[N - 2, V // 2] = float("nan")                        # a NaN: the whole row -inf (one entry for log-probs)
    x[N - 1, :V] = -float("inf")                           # an all -inf row
    lm = c.pop("lm", None)
    if lm is not None:
        l = torch.full((N, ld), float("nan"), device="cuda", dtype=BF if lm == "bf" else F32)
        w = _rand((N, V), seed + 1, 2.0, F32)
        l[:, :V] = torch.log_softmax(w, -1) if lm == "lp" else w.to(l.dtype)
        l[N - 3, 1 % V] = float("nan")                     # a NaN in the LM
        lm = l
    prev = _rand((N,), seed + 2, 5.0, F32) if c.pop("prev", False) else None
    return x, V, kind != "lp", lm, prev, c


def _check_merge(out, r, name, parity):
    got = out.to(F64)
    inf = r.out == -float("inf")
    open_eos = torch.zeros_like(inf)
    open_eos[:, 2] = r.undecided
    assert not torch.isnan(got).any(), name + ": NaN in the table"
    assert torch.equal((got == -float("inf")) & ~open_eos, inf & ~open_eos), name + ": -inf pattern differs"
    fin = ~inf & ~open_eos
    err = (got - r.out).abs()
    assert not (err[fin & (r.err == 0)] > 0).any(), name + ": inexact where the statement is exact"
    ratio = float((err / torch.where(r.err > 0, r.err, torch.ones_like(r.err)))[fin].max()) if fin.any() else 0.0
    for n in torch.nonzero(r.undecided).flatten().tolist():  # either decision, each within its bound
        g = float(got[n, 2])
        assert g == -float("inf") or abs(g - float(r.out[n, 2] if r.out[n, 2] > -float("inf") else r.eos_alt[n])) <= \
            float(r.err[n, 2])
    parity(name + " error / analytic bound", ratio, BEAM_RATIO)


@pytest.mark.parametrize("case", BM, ids=lambda c: "-".join("%s=%s" % i for i in c.items()))
def test_beam_merge(case, parity):
    N = 6
    x, V, logits, lm, prev, kw = _merge_inputs(case, N, 700 + case["V"])
    buf, out = _boxed((N, V), F32)
    from espresso_b200 import ops

    ops.beam_merge(x, V, logits, out, prev_scores=prev, lm=lm, **kw)
    torch.cuda.synchronize()
    _untouched(buf, out, "beam merge out")
    r = S.beam_merge64(x, V, logits, prev_scores=prev, lm=lm, **kw)
    _check_merge(out, r, "beam merge " + "-".join("%s=%s" % i for i in case.items()), parity)


@pytest.mark.parametrize("logits", [True, False], ids=["logits", "logprobs"])
def test_beam_merge_eos_gate_outside_bound(logits, parity):
    """Rows whose lp_eos sits 3 bounds above or below eos_factor * max: the kernel decides as float64 does."""
    N, V, f, eos = 16, 5004, 1.4, 2
    v = _rand((N, V), 800, 3.0, F32)
    x = v if logits else torch.log_softmax(v, -1)
    side = torch.where(torch.arange(N, device="cuda") % 2 == 0, 1.0, -1.0).to(F64)
    for _ in range(4):  # Newton steps on x_eos: d(margin) / d(x_eos) = 1 + (f - 1) p_eos for logits, 1 for log-probs
        r = S.beam_merge64(x, V, logits, eos_factor=f, eos=eos)
        x[:, eos] = (x.to(F64)[:, eos] + side * 3 * r.gate_err - r.gate_margin).to(F32)
    r = S.beam_merge64(x, V, logits, eos_factor=f, eos=eos)
    assert not r.undecided.any() and (r.gate_margin.abs() > r.gate_err).all()
    assert ((r.gate_margin > 0) == (side > 0)).all()
    buf, out = _boxed((N, V), F32)
    from espresso_b200 import ops

    ops.beam_merge(x, V, logits, out, eos_factor=f, eos=eos)
    torch.cuda.synchronize()
    _untouched(buf, out, "beam merge out")
    _check_merge(out, r, "beam merge eos gate %s" % ("logits" if logits else "logprobs"), parity)


# ------------------------------------------------------------------------------------------------ paths attention
@pytest.mark.parametrize("hd", [64, 96, 128])
def test_decode_self_attn_paths(hd, parity):
    H, S_, lens_l = 4, 1280, [0, 1, 31, 32, 33, 900, 1280]
    N, d = len(lens_l), 4 * hd
    q = _rand((N, d), 900 + hd)
    cache = _rand((S_, N, 2 * d), 901 + hd)
    g = torch.Generator().manual_seed(hd)
    cells = torch.zeros(S_, N, dtype=I32)
    for n, L in enumerate(lens_l):  # key i of a path lies in a later frame slot than key i - 1, in any row
        slots = torch.sort(torch.randperm(S_, generator=g)[:L]).values
        cells[:L, n] = (slots * N + torch.randint(0, N, (L,), generator=g)).to(I32)
    cells[:31, 3] = cells[:31, 2]        # hypotheses extending one another share their cells
    cells[:32, 4] = cells[:32, 3]
    cells[:900, 6] = cells[:900, 5]
    cells, lens = cells.cuda(), torch.tensor(lens_l, dtype=I32, device="cuda")
    buf, out = _boxed((N, d))
    _check(_lib().load().esp_decode_self_attn_paths(_p(q), _p(cache), _p(cells), _p(lens), S_, N, H, hd,
                                                    C.c_float(hd ** -0.5), _p(out), _stream()))
    _untouched(buf, out, "decode self paths out")
    assert (out[0] == 0).all(), "a hypothesis without keys is not exactly 0"
    ref = A.decode_self_attn_paths64(q, cache, cells, lens, H, hd ** -0.5)
    got = out.to(F64).reshape(N, H, hd)
    parity("decode self paths hd%d lens 0..1280 ctx (tau reached)" % hd,
           A.tau_reached(lambda t: bool(((got - ref.ctx64).abs() <= ref.ctx_bound(t, t)).all()), 1.0), TAU_DEC)


# ------------------------------------------------------------------------------------------------ composition
def test_joint_network_vs_float64_autograd(parity):
    """_JointFn forward and backward at a recipe-like shape against float64 autograd of the same math: LayerNorm'd
    projections, the ReLU joint and the weight-normalised fc_out, from the same bf16 inputs and parameters."""
    from test_host_orchestration import _Task
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerTransducerModelBase
    from espresso_b200.models.transformer.speech_transformer_transducer_base import _JointFn
    from espresso_b200.modules.encoder_engine import LN_EPS

    B, T, U1, J, V, d, Hd = 2, 200, 60, 512, 1000, 256, 320
    torch.manual_seed(0)
    cfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
        encoder=dict(embed_dim=d, ffn_embed_dim=512, layers=1, attention_heads=4, normalize_before=True)))
    m = SpeechTransformerTransducerModelBase.build_model(cfg, _Task(V), decoder_hidden_size=Hd, decoder_layers=1,
                                                         decoder_embed_dim=64, joint_dim=J, decoder_dropout_in=0.0,
                                                         decoder_dropout_out=0.0)
    m.finalize_(torch.device("cuda"))
    m.train()
    m.flat.zero_grad()
    enc = _rand((B, T, d), 1000).requires_grad_(True)
    dec = _rand((B, U1, Hd), 1001).requires_grad_(True)
    dl = _rand((B, T, U1, V), 1002, 1e-3)
    logits = _JointFn.apply(enc, dec, m)
    mask = logits.grad_fn.saved[10] > 0  # the kernel's own ReLU decisions (its bf16 joint activations)
    logits.backward(dl)
    torch.cuda.synchronize()
    names = ["proj_encoder.weight", "proj_encoder.bias", "laynorm_proj_encoder.weight", "laynorm_proj_encoder.bias",
             "proj_decoder.weight", "proj_decoder.bias", "laynorm_proj_decoder.weight", "laynorm_proj_decoder.bias",
             "fc_out.bias", "fc_out.weight_g", "fc_out.weight_v"]
    P = {n: m.flat.param(n).detach().to(F64).clone().requires_grad_(True) for n in names}
    e64, d64 = enc.detach().to(F64).requires_grad_(True), dec.detach().to(F64).requires_grad_(True)
    ln = torch.nn.functional.layer_norm
    pe = ln(e64 @ P["proj_encoder.weight"].t() + P["proj_encoder.bias"], (J,), P["laynorm_proj_encoder.weight"],
            P["laynorm_proj_encoder.bias"], LN_EPS)
    pd = ln(d64 @ P["proj_decoder.weight"].t() + P["proj_decoder.bias"], (J,), P["laynorm_proj_decoder.weight"],
            P["laynorm_proj_decoder.bias"], LN_EPS)
    W = P["fc_out.weight_g"] * P["fc_out.weight_v"] / P["fc_out.weight_v"].norm(dim=1, keepdim=True)
    # ReLU under the kernel's mask: where pe + pd lies within the bf16 rounding of 0 the two sides may decide
    # differently, and one flipped element moves a denc row by a whole dF term, a decision rather than a rounding error
    # (unmasked, denc reaches 3.3e-2)
    l64 = ((pe[:, :, None] + pd[:, None]) * mask) @ W.t() + P["fc_out.bias"]
    l64.backward(dl.to(F64))

    def rel(a, b):
        return float((a.detach().to(F64) - b).norm() / b.norm())

    parity("joint network logits ||err|| / ||x64||", rel(logits, l64.detach()), GRAD_REL)
    parity("joint network denc ||err|| / ||g64||", rel(enc.grad, e64.grad), GRAD_REL)
    parity("joint network ddec ||err|| / ||g64||", rel(dec.grad, d64.grad), GRAD_REL)
    for n in names:
        parity("joint network d%s ||err|| / ||g64||" % n, rel(m.flat.grad(n), P[n].grad), GRAD_REL)


# ------------------------------------------------------------------------------------------------ refusals
def test_host_refusals():
    lib = _lib()
    L = lib.load()
    e, d = _rand((1, 4, 64), 1), _rand((1, 3, 64), 2)
    fb, f = _boxed((1, 4, 3, 64))
    # misaligned vector accesses
    assert L.esp_joint_fwd(_p(e, 2), _p(d), 1, 4, 3, 64, _p(f), _stream()) != 0
    assert "16-byte aligned" in L.esp_last_error().decode()
    assert L.esp_joint_fwd(_p(e), _p(d), 1, 4, 3, 64, _p(f, 8), _stream()) != 0
    deb, de = _boxed((1, 4, 64))
    ddb, dd = _boxed((1, 3, 64), F32)
    assert L.esp_joint_bwd(_p(f, 2), _p(f), 1, 4, 3, 64, _p(de), _p(dd), _stream()) != 0
    assert "16-byte aligned" in L.esp_last_error().decode()
    assert L.esp_joint_bwd(_p(f), _p(f), 1, 4, 3, 64, _p(de, 4), _p(dd), _stream()) != 0
    # one CTA row per utterance: B beyond gridDim.y
    assert L.esp_joint_bwd(_p(f), _p(f), 65536, 1, 1, 8, _p(de), _p(dd), _stream()) != 0
    assert "at most 65535" in L.esp_last_error().decode()
    E = _rand((10, 64), 3)
    tok = torch.zeros(4, dtype=I32, device="cuda")
    xb, x = _boxed((4, 64))
    for args in ((E, 2, None, 0, x, 0), (E, 0, E, 2, x, 0), (E, 0, None, 0, x, 4)):
        assert L.esp_embed_fwd(_p(tok), _p(args[0], args[1]), _p(args[2], args[3]), 4, 64, 1.0, 4, 1, _p(args[4], args[5]),
                               0.0, 0, None, _stream()) != 0
        assert "16-byte aligned" in L.esp_last_error().decode()
    # argmax over no columns, or a row stride shorter than V
    ab, am = _boxed((4,), I32)
    assert L.esp_argmax_rows(_p(E), 64, 0, 4, _p(am), _stream()) != 0
    assert "V >= 1" in L.esp_last_error().decode()
    assert L.esp_argmax_rows(_p(E), 32, 64, 4, _p(am), _stream()) != 0
    # decode attention over more slots than the kernel's shared-memory rows
    ob, o = _boxed((2, 64))
    assert L.esp_decode_self_attn_paths(_p(E), _p(E), _p(tok), _p(tok), 1281, 2, 1, 64, C.c_float(0.125), _p(o),
                                        _stream()) != 0
    assert "slots=1281" in L.esp_last_error().decode()
    torch.cuda.synchronize()
    for b, what in ((fb, "joint out"), (deb, "denc"), (ddb, "ddec"), (xb, "embed x"), (ab, "argmax out"), (ob, "paths out")):
        _untouched(b, b[:0], "refused " + what)
