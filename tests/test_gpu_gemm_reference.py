"""The wgmma GEMM (espresso_b200/csrc/gemm_tcgen05.cu) and its implicit-GEMM 3x3 convolutions against the float64
statement in oracle/gemm64.py, per element:

    |c - c64| <= TAU * mag                       fp32 outputs (mag = |A| |B|^T carried through the epilogue)
    |c - c64| <= TAU * mag + 2^-8 |c64|          bf16 outputs (one rounding of the fp32 result)
    ... + EPS_SIG * apx                          SiLU / SiLU' epilogues (tanh.approx.f32 sigmoid)

TAU is a few fp32 roundings of the reduction; one bf16 rounding of the accumulator, of a split-K partial or of an fp32
residual costs up to 2^-9 of mag, far above it, so every such mistake fails here (non-negative inputs make mag = |c64|
and leave it nowhere to hide).  Every case writes its achieved error next to the bound with the `parity` fixture.

Sections: (a) every template instance (tile width x multicast x operand majors) at ragged M / N / K, (b) exact gathers
through selection matrices, (c) bit-exact consistency between outputs of the same call, (d) every epilogue branch,
(e) misaligned store paths and NaN-payload sentinels around every output, (f) the product's call forms at recipe shapes,
(g) split-K accumulate and the fused bias-gradient row sums, (h) the three convolutions, (i) clean host refusals."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32

# Bounds, set at 3-4x the largest error reached on an NVIDIA H100 80GB HBM3 (400 W power limit); every run writes the
# values reached to the parity report.  Reached: 2.3e-6 (non-negative inputs, K = 1000), 3.1e-7 (randn), 6.4e-7 (split-K
# accumulate, K up to 20 000), 6.6e-9 (row sums), 2.5e-7 (convolutions).  The fp32 outputs of all 20 instances are
# bit-identical.
TAU = 8e-6            # fp32 GEMM / conv results, per element against the magnitude
TAU_ACC = 2.5e-6      # split-K accumulate (atomic order varies between runs) and the bias-gradient row sums
EPS_SIG = 2.5e-4      # |sigmoid~ - sigmoid| of fast_sigmoid: 0.5 * |tanh.approx.f32 error| (PTX: 2^-10.987) + roundings
BF16_REL = 2.0 ** -8  # one bf16 rounding of the fp32 result (half an ulp is 2^-8 of the value at most; plus a flip)

SENT16 = 0x7FA5        # NaN payloads that no kernel ever produces
SENT32 = 0x7FC0DEAD

INSTANCES = [(64, 1), (128, 1), (128, 2), (256, 1), (256, 2)]  # (tile width BN, CTAs per cluster MC)
MAJORS = [(True, True), (True, False), (False, True), (False, False)]  # (A K-major, B K-major)


@pytest.fixture(scope="module", autouse=True)
def _env():
    from espresso_b200 import ops

    assert torch.cuda.is_available()
    assert not os.environ.get("ESP_GEMM_MULTICAST", "").startswith("0"), \
        "ESP_GEMM_MULTICAST=0 runs every 2-CTA cluster instance as MC 1: unset it to test the multicast instances"
    saved = ops._SEED_T
    ops.set_seed_tensor(None)  # dropout masks of these tests depend on the call's seed alone
    yield
    ops.set_seed_tensor(saved)


def _ops():
    from espresso_b200 import ops

    return ops


def _g64():
    from oracle import gemm64

    return gemm64


def _r8(n):
    return (n + 7) // 8 * 8


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _instance(M, N, tile_n, accumulate=False):
    """(BN, MC) the host picks (esp_gemm_bf16): tile_n 64/128/256 forces the width, 512 forces 256-wide 2-CTA clusters;
    128- and 256-wide tiles pair M tiles when their count is even or at least 16."""
    tm = -(-M // 128)
    if tile_n == 512:
        return 256, 2
    bn = tile_n if tile_n in (64, 128, 256) else (128 if N > 64 else 64)
    assert tile_n or accumulate
    return bn, (2 if bn >= 128 and (tm % 2 == 0 or tm >= 16) else 1)


def _ksplit(M, N, K):
    """K splits of an accumulating GEMM (esp_gemm_bf16): best utilisation of the SMs, >= 4 k-blocks per split."""
    bn = 128 if N > 64 else 64
    t = -(-M // 128) * -(-N // bn)
    num_kb = -(-K // 64)
    best, ks_best = -1.0, 1
    ks = 1
    while ks <= max(num_kb // 4, 1) and (ks - 1) * t < _sms():
        items = t * ks
        e = items / (-(-items // _sms()) * _sms()) - 0.01 * ks
        if e > best:
            best, ks_best = e, ks
        ks += 1
    return ks_best


def _rand(shape, fam, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand(shape, generator=g, device="cuda") if fam == "uniform" else torch.randn(shape, generator=g, device="cuda")
    return (x * scale).to(BF)


def _store(x, kmajor, pad=8):
    """x [rows, k] as a GEMM operand: K-major rows of ld k + pad, or MN-major [k, ld] with ld = r8(rows) + pad; the
    padding holds NaN, so a kernel that reads past the logical extent poisons its result."""
    rows, k = x.shape
    if kmajor:
        buf = torch.full((rows, k + pad), float("nan"), device=x.device, dtype=BF)
        buf[:, :k] = x
        return buf, k + pad
    ld = _r8(rows) + pad
    buf = torch.full((k, ld), float("nan"), device=x.device, dtype=BF)
    buf[:, :rows] = x.t()
    return buf, ld


def _sentinel(shape, dtype):
    t = torch.empty(shape, device="cuda", dtype=dtype)
    t.view(torch.int16 if dtype == BF else torch.int32).fill_(SENT16 if dtype == BF else SENT32)
    return t


def _logical(C, M, N, ldc, nb1=1, nb2=1, sC=(0, 0)):
    return C.as_strided((nb2, nb1, M, N), (sC[1], sC[0], ldc, 1))


def _assert_untouched(buf, view, what):
    """Every element of `buf` outside the logical output `view` (a strided view into buf's storage) still holds the
    sentinel."""
    flat = buf.reshape(-1)
    mark = torch.zeros(flat.numel(), dtype=torch.bool, device=buf.device)
    idx = torch.arange(flat.numel(), device=buf.device)
    off = view.storage_offset() - buf.storage_offset()
    mark[idx.as_strided(view.shape, view.stride(), off).reshape(-1)] = True
    bits = flat.view(torch.int16 if buf.dtype == BF else torch.int32)
    pat = SENT16 if buf.dtype == BF else SENT32
    bad = (~mark) & (bits != pat)
    assert not bad.any(), "%s: %d elements written outside the logical output (first at %d)" % (
        what, int(bad.sum()), int(bad.nonzero()[0]))


def _achieved(c, ref, *, bf16):
    """_tau_reached for the output of a gemm64 result."""
    return _tau_reached(c, ref.c, ref.mag, ref.apx, bf16=bf16)


def _achieved_c2(c2, ref):
    return _tau_reached(c2, ref.c2, ref.mag2, None, bf16=True)


def _tau_reached(c, v, m, a, *, bf16, apx_eps=EPS_SIG):
    """Smallest tau with |c - c64| <= tau * mag + 2^-8 |c64| [bf16] + apx_eps * apx; elements of zero magnitude must be
    exact (up to the other terms)."""
    c = c.double()
    assert torch.isfinite(c).all(), "non-finite output"
    extra = torch.zeros_like(v)
    if bf16:
        extra = extra + BF16_REL * v.abs()
    if a is not None:
        extra = extra + apx_eps * a
    ex = (c - v).abs() - extra
    zero = m == 0
    assert not (ex[zero] > 0).any(), "non-zero error where the magnitude is 0"
    return float((ex.clamp_min(0) / torch.where(zero, torch.ones_like(m), m)).max()) if ex.numel() else 0.0


def _sig_achieved(c, ref, tau, bf16):
    """Smallest eps with |c - c64| <= tau * mag + 2^-8 |c64| [bf16] + eps * apx over the elements with apx > 0."""
    c = c.double()
    ex = (c - ref.c).abs() - tau * ref.mag - (BF16_REL * ref.c.abs() if bf16 else 0)
    sel = ref.apx > 0
    return float((ex[sel].clamp_min(0) / ref.apx[sel]).max()) if sel.any() else 0.0


def _pair(A, B, C, M, N, K, lda, ldb, ldc, **kw):
    """float64 statement first (it reads the accumulate target before the kernel adds to it), then the kernel."""
    ref = _g64().gemm(A, B, C, M, N, K, lda, ldb, ldc, **kw)
    _ops().gemm(A, B, C, M, N, K, lda, ldb, ldc, **kw)
    return _logical(C, M, N, ldc, kw.get("nb1", 1), kw.get("nb2", 1), kw.get("sC", (0, 0))), ref


# ------------------------------------------------------------------------------------------ (a) every template instance
def _shapes(bn, mc):
    """tile_n reaching (bn, mc) and the shapes: ragged M (3 or 4 tiles; 17 tiles / 3 tiles for the pair's missing odd
    tile), N with N mod 32 != 0 and N mod BN != 0, K = 8, 40 (< one 64-block), 200 and 1000 (partial last block)."""
    N = {64: 200, 128: 328, 256: 520}[bn]
    M = 300 if mc == 1 else 500
    tile_n = 512 if (bn, mc) == (256, 2) else bn
    shapes = [(M, N, K) for K in (8, 40, 200, 1000)]
    if mc == 2:
        shapes.append((2100 if bn == 128 else 300, N, 136))
    return tile_n, shapes


def _operands(M, N, K, ak, bk, fam, seed):
    a, b = _rand((M, K), fam, seed), _rand((N, K), fam, seed + 1)
    A, lda = _store(a, ak)
    Bm, ldb = _store(b, bk)
    return a, b, A, lda, Bm, ldb


@pytest.mark.parametrize("ak,bk", MAJORS)
@pytest.mark.parametrize("bn,mc", INSTANCES)
def test_instance_vs_float64(bn, mc, ak, bk, parity):
    tile_n, shapes = _shapes(bn, mc)
    worst = {"uniform": 0.0, "randn": 0.0}
    for M, N, K in shapes:
        assert _instance(M, N, tile_n) == (bn, mc)
        for fam in worst:
            a, b, A, lda, Bm, ldb = _operands(M, N, K, ak, bk, fam, M + N + K)
            ldc = N + 8
            c32 = _sentinel((M + 2, ldc), F32)
            c16 = _sentinel((M + 2, ldc), BF)
            kw = dict(a_kmajor=ak, b_kmajor=bk, tile_n=tile_n)
            out32, ref = _pair(A, Bm, c32, M, N, K, lda, ldb, ldc, **kw)
            out16, _ = _pair(A, Bm, c16, M, N, K, lda, ldb, ldc, **kw)
            torch.cuda.synchronize()
            _assert_untouched(c32, out32, "fp32 C")
            _assert_untouched(c16, out16, "bf16 C")
            # (c) the bf16 output of a call is its fp32 output rounded to nearest-even
            assert torch.equal(out16, out32.to(BF)), "bf16 output != RN(fp32 output), K=%d %s" % (K, fam)
            worst[fam] = max(worst[fam], _achieved(out32, ref, bf16=False))
    for fam, w in worst.items():
        parity("gemm BN%d MC%d A%s B%s %s inputs, ragged M/N/K (err / |A||B|^T)" % (
            bn, mc, "k" if ak else "mn", "k" if bk else "mn", fam), w, TAU)


# ------------------------------------------------------------------------------------------ (b) exact gathers
@pytest.mark.parametrize("side", ["A", "B"])
@pytest.mark.parametrize("ak,bk", MAJORS)
@pytest.mark.parametrize("bn,mc", INSTANCES)
def test_selection_gather_is_exact(bn, mc, ak, bk, side):
    """A (or B) holds one 1.0 per row at column m mod K (n mod K): the rows cover every k of every k16 step, every 64-block
    boundary and the partial tail block, so C must be the selected columns of the other operand bit for bit."""
    tile_n, shapes = _shapes(bn, mc)
    M, N, _ = shapes[0]
    K = 200
    assert _instance(M, N, tile_n) == (bn, mc)
    dev = torch.device("cuda")
    a, b = _rand((M, K), "randn", 5), _rand((N, K), "randn", 6)
    if side == "A":
        a = torch.zeros(M, K, device=dev, dtype=BF)
        a[torch.arange(M), torch.arange(M) % K] = 1
        want = b[:, torch.arange(M, device=dev) % K].t()
    else:
        b = torch.zeros(N, K, device=dev, dtype=BF)
        b[torch.arange(N), torch.arange(N) % K] = 1
        want = a[:, torch.arange(N, device=dev) % K]
    A, lda = _store(a, ak)
    Bm, ldb = _store(b, bk)
    for dt in (F32, BF):
        c = _sentinel((M, N + 8), dt)
        _ops().gemm(A, Bm, c, M, N, K, lda, ldb, N + 8, a_kmajor=ak, b_kmajor=bk, tile_n=tile_n)
        assert torch.equal(c[:, :N], want.to(dt)), "gather through %s, %s output" % (side, dt)
        _assert_untouched(c, c[:, :N], "gather output")


# ------------------------------------------------------------------------------------------ (c) consistency
def test_fp32_outputs_bit_identical_across_instances(parity):
    """Each output element sums its k products in the same order (64-blocks in order, k16 steps in order) whatever the
    tile width, multicast and operand majors: the fp32 results of all 20 instances agree bit for bit."""
    N, Mmax = 520, 500
    for K, fam in ((1000, "randn"), (200, "uniform")):
        a, b = _rand((Mmax, K), fam, 11), _rand((N, K), fam, 12)
        outs = []
        for bn, mc in INSTANCES:
            tile_n, shapes = _shapes(bn, mc)
            M = shapes[0][0]
            assert _instance(M, N, tile_n) == (bn, mc)
            for ak, bk in MAJORS:
                A, lda = _store(a[:M], ak)
                Bm, ldb = _store(b, bk)
                c = torch.empty(M, N, device="cuda", dtype=F32)
                _ops().gemm(A, Bm, c, M, N, K, lda, ldb, N, a_kmajor=ak, b_kmajor=bk, tile_n=tile_n)
                outs.append(c[:300])
        diff = max(float((o - outs[0]).abs().max()) for o in outs)
        parity("fp32 output, max |difference| between the 20 instances, K=%d %s" % (K, fam), diff, 0.0)


# ------------------------------------------------------------------------------------------ (d) epilogue branches
BRANCHES = {
    "bias": dict(bias=True),
    "c2": dict(bias=True, C2=True),
    "relu": dict(bias=True, act=1),
    "silu": dict(bias=True, act=2),
    "relu_bwd": dict(act=3),
    "silu_bwd": dict(act=4),
    "dropout1": dict(drop_mode=1),
    "dropout2": dict(drop_mode=2),
    "alpha": dict(alpha=-0.625),
    "resid_bf16": dict(R=BF, beta=0.75),
    "resid_fp32": dict(R=F32, beta=-1.25),
    "ffn1": dict(bias=True, act=2, C2=True, drop_mode=1),
    "ffn2": dict(bias=True, drop_mode=1, alpha=0.5, R=BF, beta=1.0),
    "dgrad_relu": dict(act=3, drop_mode=2, alpha=1.5, R=F32, beta=0.5),
    "dgrad_silu": dict(act=4, drop_mode=2, C2=True, bias=True, R=BF, beta=-2.0),
}


def _epilogue_kw(spec, M, N, seed):
    kw = {}
    if spec.get("bias"):
        kw["bias"] = _rand((N,), "randn", seed + 1)
    if spec.get("act"):
        kw["act"] = spec["act"]
    if spec.get("act") in (3, 4):
        ld = N + 24
        aux = _rand((M, ld), "randn", seed + 2, 2.0)
        aux[::3, ::4] = 0  # ReLU' passes nothing at aux == 0 exactly
        kw.update(aux=aux, ld_aux=ld)
    if spec.get("drop_mode"):
        kw.update(drop_p=0.25, drop_mode=spec["drop_mode"], seed=4321 + seed)
    if "alpha" in spec:
        kw["alpha"] = spec["alpha"]
    if spec.get("R") is not None:
        ld = N + 16
        r = _rand((M, ld), "randn", seed + 3).to(spec["R"])
        if spec["R"] == F32:
            r = r + 1e-3 * torch.randn(M, ld, device="cuda")  # not representable in bf16
        kw.update(R=r, ldr=ld, beta=spec["beta"])
    return kw


@pytest.mark.parametrize("tile_n", [64, 0, 512])
@pytest.mark.parametrize("dt", [F32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("branch", list(BRANCHES))
def test_epilogue_branch(branch, dt, tile_n, parity):
    """M = 300 (3 tiles), N = 200 (a valid < 32 tail chunk), K = 200; randn and non-negative operands."""
    spec = BRANCHES[branch]
    M, N, K = 300, 200, 200
    worst, worst_sig = 0.0, 0.0
    for fam in ("randn", "uniform"):
        seed = 100 + len(branch) + (fam == "uniform")
        a, b = _rand((M, K), fam, seed), _rand((N, K), fam, seed + 7, 0.1)
        A, lda = _store(a, True)
        Bm, ldb = _store(b, True)
        kw = _epilogue_kw(spec, M, N, seed)
        ldc = N + 8
        c = _sentinel((M + 1, ldc), dt)
        c2 = _sentinel((M + 1, ldc), BF) if spec.get("C2") else None
        out, ref = _pair(A, Bm, c, M, N, K, lda, ldb, ldc, tile_n=tile_n, C2=c2, **kw)
        torch.cuda.synchronize()
        _assert_untouched(c, out, "C")
        worst = max(worst, _achieved(out, ref, bf16=dt == BF))
        if spec.get("act") in (2, 4):
            worst_sig = max(worst_sig, _sig_achieved(out, ref, TAU, dt == BF))
        if c2 is not None:
            o2 = _logical(c2, M, N, ldc)
            _assert_untouched(c2, o2, "C2")
            worst = max(worst, _achieved_c2(o2, ref))
            # (c) C2 is bf16(acc + bias): the fp32 output of the same GEMM with the bias alone, rounded
            c32 = torch.empty(M, N, device="cuda", dtype=F32)
            _ops().gemm(A, Bm, c32, M, N, K, lda, ldb, N, tile_n=tile_n, bias=kw.get("bias"))
            assert torch.equal(o2[0, 0], c32.to(BF)), "C2 != bf16(acc + bias)"
    name = "epilogue %-10s %s out, tile_n %d" % (branch, "fp32" if dt == F32 else "bf16", tile_n)
    parity(name + " (err / mag)", worst, TAU)
    if spec.get("act") in (2, 4):
        parity(name + " (sigmoid approximation error)", worst_sig, EPS_SIG)


@pytest.mark.parametrize("dt", [F32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("roff", [0, 1])
@pytest.mark.parametrize("T", [37, 70, 30])
def test_skew_residual(T, roff, dt, parity):
    """Scores with the fused Transformer-XL skew: R = BD[m, (T-1) - m + n]; 2T-1 is not a multiple of 8, and the BD view
    starts on an even or an odd element (the funnel-shift path for the upper half of a word; T = 30: tail path only)."""
    H, Bz, hd = 2, 3, 64
    d = H * hd
    q, k = _rand((Bz * T, d), "randn", T), _rand((Bz * T, d), "randn", T + 1)
    ldp, ldt = _r8(2 * T - 1), _r8(T)
    store = torch.full((H * Bz * T * ldp + 8,), float("nan"), device="cuda", dtype=BF)
    bd = store[roff:roff + H * Bz * T * ldp].view(H, Bz, T, ldp)
    bd[..., : 2 * T - 1] = _rand((H, Bz, T, 2 * T - 1), "randn", T + 2)
    S = _sentinel((H, Bz, T, ldt), dt)
    out, ref = _pair(q, k, S, T, T, hd, d, d, ldt, nb1=H, nb2=Bz, sA=(hd, T * d), sB=(hd, T * d),
                     sC=(Bz * T * ldt, T * ldt), R=bd, ldr=ldp, sR=(Bz * T * ldp, T * ldp), skew_r=T, alpha=0.125)
    torch.cuda.synchronize()
    _assert_untouched(S, out, "scores")
    parity("skew T'=%d, BD offset %d, %s out (err / mag)" % (T, roff, "fp32" if dt == F32 else "bf16"),
           _achieved(out, ref, bf16=dt == BF), TAU)


# ------------------------------------------------------------------------------------------ (e) store paths, sentinels
STORES = ["f32_ldc_mod4", "f32_offset", "bf16_ldc_mod8", "bf16_offset", "batched_gaps_f32", "batched_gaps_bf16"]


@pytest.mark.parametrize("tile_n", [64, 0, 512])
@pytest.mark.parametrize("case", STORES)
def test_store_paths_and_sentinels(case, tile_n, parity):
    """Scalar store / load paths for rows whose base is not 16-byte aligned (ldc mod 4 != 0 in fp32, ldc mod 8 != 0 in
    bf16, column-offset views) with C2, a misaligned bf16 residual and aux; batched outputs with gaps between batch
    strides.  Nothing outside the logical [nb2, nb1, M, N] of C and C2 may change."""
    M, N, K = 300, 200, 136
    nb1, nb2 = (2, 3) if case.startswith("batched") else (1, 1)
    dt = F32 if "f32" in case else BF
    a = _rand((nb2 * nb1 * M, K), "randn", 21)
    b = _rand((nb1 * N, K), "randn", 22, 0.1)  # broadcast over nb2
    kw = dict(tile_n=tile_n, nb1=nb1, nb2=nb2, sA=(M * K, nb1 * M * K), sB=(N * K, 0))
    if case == "f32_ldc_mod4":
        ldc, off, ext = N + 2, 0, (M + 1) * (N + 2)
    elif case == "bf16_ldc_mod8":
        ldc, off, ext = N + 3, 0, (M + 1) * (N + 3)
    elif case.endswith("offset"):
        ldc, off, ext = N + 16, 3 if dt == BF else 1, (M + 1) * (N + 16)
    else:
        ldc, off = N + 8, 0
        s1 = M * ldc + 24
        s2 = nb1 * s1 + 40
        ext = nb2 * s2 + 16
        kw["sC"] = (s1, s2)
    cbuf = _sentinel((ext,), dt)
    c2buf = _sentinel((ext,), BF)
    C, C2 = cbuf[off:], c2buf[off:]
    lr = N + 5  # bf16 residual rows start on odd elements
    rbuf = _rand((nb2 * nb1 * M * lr + 1,), "randn", 23)
    aux = _rand((nb2 * nb1 * M * (N + 1),), "randn", 24)
    aux[::7] = 0
    kw.update(bias=_rand((N,), "randn", 25), C2=C2, act=3, aux=aux, ld_aux=N + 1, sAux=(M * (N + 1), nb1 * M * (N + 1)),
              R=rbuf[1:], ldr=lr, sR=(M * lr, nb1 * M * lr), beta=0.5, alpha=-1.5)
    out, ref = _pair(a, b, C, M, N, K, K, K, ldc, **kw)
    torch.cuda.synchronize()
    _assert_untouched(cbuf, out, "C (%s)" % case)
    o2 = _logical(C2, M, N, ldc, nb1, nb2, kw.get("sC", (0, 0)))
    _assert_untouched(c2buf, o2, "C2 (%s)" % case)
    w = max(_achieved(out, ref, bf16=dt == BF), _achieved_c2(o2, ref))
    parity("store path %s, tile_n %d (err / mag)" % (case, tile_n), w, TAU)


def test_fp32_residual_store_offsets(parity):
    """fp32 residual whose rows start off 16-byte alignment, fp32 output through a column-offset view."""
    M, N, K = 260, 136, 72
    a, b = _rand((M, K), "uniform", 31), _rand((N, K), "uniform", 32)
    r = torch.rand(M * (N + 3) + 1, device="cuda") + 1e-3
    cbuf = _sentinel((M, N + 9), F32)
    C = cbuf[:, 1:]
    out, ref = _pair(a, b, C, M, N, K, K, K, N + 9, R=r[1:], ldr=N + 3, beta=0.375)
    torch.cuda.synchronize()
    _assert_untouched(cbuf, out, "C")
    parity("fp32 residual at odd offsets, fp32 out at a column offset (err / mag)", _achieved(out, ref, bf16=False), TAU)


# ------------------------------------------------------------------------------------------ (f) recipe call forms
RECIPE_T = [25, 250, 407, 875]
FORMS = ["qkv", "ffn1", "ffn2", "out_proj", "dgrad_silu", "dgrad_relu", "bd_per_head", "bd_shared", "scores_skew",
         "pv", "dv", "dk", "dq_v", "dpos_splitk", "output_proj"]


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("T", RECIPE_T)
def test_recipe_call_forms(T, form, parity):
    """The GEMM calls of encoder_engine.py / decoder_engine.py, argument for argument, at d = 512, FFN 2048, H = 8,
    hd = 64, V = 5004 and encoder lengths T' of the recipes (about 3500 rows per batch)."""
    ops = _ops()
    d, Fd, H, hd, V = 512, 2048, 8, 64, 5004
    Bz = max(1, 3500 // T)
    R = Bz * T
    ldt, ldp = _r8(T), _r8(2 * T - 1)
    s = T + len(form)
    x = _rand((R, d), "randn", s)
    W = lambda n, k, i: _rand((n, k), "randn", s + i, k ** -0.5)  # noqa: E731
    bias = lambda n, i: _rand((n,), "randn", s + i, 0.1)  # noqa: E731
    fp32 = False
    if form == "qkv":
        y = torch.empty(R, 3 * d, device="cuda", dtype=BF)
        out, ref = _pair(x, W(3 * d, d, 1), y, R, 3 * d, d, d, d, 3 * d, bias=bias(3 * d, 2))
    elif form == "ffn1":
        y = torch.empty(R, Fd, device="cuda", dtype=BF)
        U = torch.empty(R, Fd, device="cuda", dtype=BF)
        out, ref = _pair(x, W(Fd, d, 1), y, R, Fd, d, d, d, Fd, bias=bias(Fd, 2), act=2, C2=U, drop_p=0.1, drop_mode=1,
                         seed=s)
        parity("recipe ffn1 C2 T'=%d (err / mag)" % T,
               _achieved_c2(_logical(U, R, Fd, Fd), ref), TAU)
    elif form in ("ffn2", "out_proj"):
        k = Fd if form == "ffn2" else d
        h = _rand((R, k), "randn", s + 3, 0.5)
        y = torch.empty(R, d, device="cuda", dtype=BF)
        out, ref = _pair(h, W(d, k, 1), y, R, d, k, k, k, d, bias=bias(d, 2), drop_p=0.1, drop_mode=1, seed=s,
                         alpha=0.5 if form == "ffn2" else 1.0, R=x, ldr=d, beta=1.0)
    elif form.startswith("dgrad"):
        dZ = _rand((R, d), "randn", s + 4)
        U = _rand((R, Fd), "randn", s + 5, 2.0)
        U[::5, ::3] = 0
        y = torch.empty(R, Fd, device="cuda", dtype=BF)
        W2 = W(d, Fd, 1)
        out, ref = _pair(dZ, W2, y, R, Fd, d, d, Fd, Fd, b_kmajor=False, act=4 if form == "dgrad_silu" else 3, aux=U,
                         ld_aux=Fd, drop_p=0.1, drop_mode=2, seed=s)
    elif form.startswith("bd"):
        qv = _rand((R, d), "randn", s + 6, 0.3)
        E = d if form == "bd_per_head" else hd
        Pp = _rand((2 * T - 1, E), "randn", s + 7)
        ph = hd if E == d else 0
        BD = _sentinel((H, Bz, T, ldp), BF)
        out, ref = _pair(qv, Pp, BD, T, 2 * T - 1, hd, d, E, ldp, nb1=H, nb2=Bz, sA=(hd, T * d), sB=(ph, 0),
                         sC=(Bz * T * ldp, T * ldp))
        torch.cuda.synchronize()
        _assert_untouched(BD, out, "BD")
    elif form == "scores_skew":
        qu = _rand((R, d), "randn", s + 6, 0.3)
        qkv = _rand((R, 3 * d), "randn", s + 8)
        BD = torch.full((H, Bz, T, ldp), float("nan"), device="cuda", dtype=BF)
        BD[..., : 2 * T - 1] = _rand((H, Bz, T, 2 * T - 1), "randn", s + 9)
        S = _sentinel((H, Bz, T, ldt), BF)
        out, ref = _pair(qu, qkv[:, d:], S, T, T, hd, d, 3 * d, ldt, nb1=H, nb2=Bz, sA=(hd, T * d), sB=(hd, T * 3 * d),
                         sC=(Bz * T * ldt, T * ldt), R=BD, ldr=ldp, sR=(Bz * T * ldp, T * ldp), skew_r=T)
        torch.cuda.synchronize()
        _assert_untouched(S, out, "scores")
    elif form in ("pv", "dv", "dk"):
        P = torch.full((H, Bz, T, ldt), float("nan"), device="cuda", dtype=BF)
        P[..., :T] = _rand((H, Bz, T, T), "uniform", s + 10, 2.0 / T)
        if form == "pv":
            qkv = _rand((R, 3 * d), "randn", s + 8)
            ctx = _sentinel((R, d), BF)
            out, ref = _pair(P, qkv[:, 2 * d:], ctx, T, hd, T, ldt, 3 * d, d, b_kmajor=False, nb1=H, nb2=Bz,
                             sA=(Bz * T * ldt, T * ldt), sB=(hd, T * 3 * d), sC=(hd, T * d))
        else:
            g = _rand((R, d), "randn", s + 11)
            dqkv = _sentinel((R, 3 * d), BF)
            dst = dqkv[:, 2 * d:] if form == "dv" else dqkv[:, d:2 * d]
            out, ref = _pair(P, g, dst, T, hd, T, ldt, d, 3 * d, a_kmajor=False, b_kmajor=False, nb1=H, nb2=Bz,
                             sA=(Bz * T * ldt, T * ldt), sB=(hd, T * d), sC=(hd, T * 3 * d))
            torch.cuda.synchronize()
            _assert_untouched(dqkv, out, "dqkv")
    elif form in ("dq_v", "dpos_splitk"):
        dBD = torch.full((H, Bz, T, ldp), float("nan"), device="cuda", dtype=BF)
        dBD[..., : 2 * T - 1] = _rand((H, Bz, T, 2 * T - 1), "randn", s + 12, 0.05)
        if form == "dq_v":
            Pp = _rand((2 * T - 1, d), "randn", s + 7)
            dqv = _sentinel((R, d), BF)
            out, ref = _pair(dBD, Pp, dqv, R, hd, 2 * T - 1, ldp, d, d, b_kmajor=False, nb1=H, nb2=1,
                             sA=(Bz * T * ldp, 0), sB=(hd, 0), sC=(hd, 0))
        else:
            qv = _rand((R, d), "randn", s + 6, 0.3)
            dP = torch.zeros(2 * T - 1, d, device="cuda", dtype=F32)
            out, ref = _pair(dBD, qv, dP, 2 * T - 1, hd, R, ldp, d, d, a_kmajor=False, b_kmajor=False, nb1=H, nb2=1,
                             sA=(Bz * T * ldp, 0), sB=(hd, 0), sC=(hd, 0), accumulate=True)
            fp32 = True
    elif form == "output_proj":
        ldV = _r8(V)
        logits = torch.zeros(R, ldV, device="cuda", dtype=BF)
        out, ref = _pair(x, W(V, d, 1), logits, R, V, d, d, d, ldV, bias=bias(V, 2))
        torch.cuda.synchronize()
        assert not logits[:, V:].any(), "padding columns of the logits written"
    torch.cuda.synchronize()
    parity("recipe %-12s T'=%d (err / mag)" % (form, T), _achieved(out, ref, bf16=not fp32),
           TAU_ACC if form == "dpos_splitk" else TAU)


# ------------------------------------------------------------------------------------------ (g) accumulate, split-K
WGRAD = [
    # out rows M, out cols N, reduction rows K, rowsum_scale, alpha
    (100, 64, 3001, 1.0, 1.0),     # BN 64, 1 part, MC 1
    (300, 200, 3001, 0.5, 1.0),    # 2 N tiles share the row sums, MC 1
    (260, 600, 20000, 1.0, 1.0),   # 4 parts, MC 1, split K
    (500, 200, 20000, -2.0, 1.0),  # 2 parts, MC 2 (4 M tiles), split K
    (1000, 520, 9000, 0.25, -1.0),  # 4 parts, MC 2, alpha = -1
    (512, 2048, 20000, 1.0, 1.0),  # FFN1 weight gradient (linear_wgrad form)
]


@pytest.mark.parametrize("case", WGRAD)
def test_wgrad_accumulate_and_rowsum(case, parity):
    """C (fp32) += alpha * A^T B with both operands MN-major (A = dy^T), split-K vector reductions, and the bias gradient
    rowsum_a += rowsum_scale * sum_k A from the same launch; M mod 8 != 0 for the row guard."""
    M, N, K, rs_scale, alpha = case
    bn, mc = _instance(M, N, 0, accumulate=True)
    parts = 4 if -(-N // bn) >= 4 else (2 if -(-N // bn) >= 2 else 1)
    ks = _ksplit(M, N, K)
    assert K < 10000 or ks > 1
    dy = _rand((K, M), "randn", M + K)
    xx = _rand((K, N), "randn", M + K + 1)
    A, lda = _store(dy.t(), False)
    Bm, ldb = _store(xx.t(), False)
    C = torch.randn(M, N, device="cuda")
    gb = torch.randn(M + 5, device="cuda")
    tail = gb[M:].clone()
    out, ref = _pair(A, Bm, C, M, N, K, lda, ldb, N, a_kmajor=False, b_kmajor=False, accumulate=True, alpha=alpha,
                     rowsum_a=gb, rowsum_scale=rs_scale)
    torch.cuda.synchronize()
    assert torch.equal(gb[M:], tail), "row sums written past M"
    name = "wgrad M=%d N=%d K=%d (BN%d MC%d, %d parts, ksplit %d)" % (M, N, K, bn, mc, parts, ks)
    parity(name + " C (err / mag)", _achieved(out, ref, bf16=False), TAU_ACC)
    rs = gb[:M].double()
    parity(name + " row sums (err / mag)", float(((rs - ref.rowsum).abs() / ref.rowsum_mag).max()), TAU_ACC)


def test_linear_wgrad_recipe(parity):
    """ops.linear_wgrad at 20 000 rows (split K) into the flat-buffer form gW [N, K] with the bias gradient."""
    ops = _ops()
    rows, N, K = 20000, 512, 512
    dy, x = _rand((rows, N), "randn", 41), _rand((rows, K), "uniform", 42)
    gW = torch.randn(N * K, device="cuda")
    gb = torch.randn(N, device="cuda")
    ref = _g64().gemm(dy, x, gW.view(N, K), N, K, rows, N, K, K, a_kmajor=False, b_kmajor=False, accumulate=True,
                      rowsum_a=gb)
    assert _ksplit(N, K, rows) > 1
    ops.linear_wgrad(dy, x, gW, gb)
    torch.cuda.synchronize()
    parity("linear_wgrad 20000 x 512 x 512 (err / mag)", _achieved(gW.view(1, 1, N, K), ref, bf16=False), TAU_ACC)
    parity("linear_wgrad bias gradient (err / mag)", float(((gb.double() - ref.rowsum).abs() / ref.rowsum_mag).max()),
           TAU_ACC)


# ------------------------------------------------------------------------------------------ (h) convolutions
CONV = [
    # B, T, F, Cin, Cout, stride
    (2, 37, 64, 64, 64, (1, 1)),    # forward box bf = 16
    (2, 40, 16, 128, 128, (2, 2)),  # bf = 8, 128-wide tiles
    (1, 50, 12, 64, 128, (1, 1)),   # bf = 4
    (2, 21, 6, 128, 64, (1, 1)),    # bf = 2
    (1, 33, 5, 64, 64, (1, 2)),     # bf = 1 (forward F' = 3), odd F with stride 2
    (2, 19, 83, 64, 64, (2, 1)),    # odd T with stride 2
    (1, 1, 1, 64, 64, (1, 1)),      # every tap but the centre out of bounds
    (1, 2, 3, 64, 128, (2, 2)),     # empty parity classes of the input gradient
    (1, 3, 2, 128, 64, (1, 2)),
    (1, 3, 3, 64, 64, (2, 1)),
    (2, 100, 40, 64, 64, (2, 2)),   # weight gradient split over K; Cin = 64: an all-out-of-bounds tap chunk
    (1, 3500, 80, 64, 64, (2, 2)),  # 80-dim fbank, 35 s: the stride-2 64 -> 64 layer of the conv front end
    (1, 1750, 40, 64, 128, (1, 1)),
]


@pytest.mark.parametrize("case", CONV, ids=lambda c: "B%d_T%d_F%d_%dto%d_s%d%d" % (c[:5] + c[5]))
def test_conv3x3_vs_float64(case, parity):
    ops, g64 = _ops(), _g64()
    B, T, Fq, Cin, Cout, stride = case
    x = _rand((B, T, Fq, Cin), "randn", T + Fq)
    w = _rand((Cout, 3, 3, Cin), "randn", T + Fq + 1, (9 * Cin) ** -0.5)
    y = ops.conv3x3_fwd(x, w, stride)
    y64, ymag = g64.conv3x3_fwd(x, w, stride)
    dy = _rand(tuple(y.shape), "randn", T + Fq + 2)
    dx = ops.conv3x3_dgrad(dy, w, x.shape, stride)
    dx64, dxmag = g64.conv3x3_dgrad(dy, w, x.shape, stride)
    dw = torch.randn(Cout, 3, 3, Cin, device="cuda")
    dw64, dwmag = g64.conv3x3_wgrad(dy, x, stride, dw)
    ops.conv3x3_wgrad(dy, x, dw, stride)
    torch.cuda.synchronize()
    name = "conv3x3 B%d T%d F%d %d->%d stride %s" % (B, T, Fq, Cin, Cout, stride)
    parity(name + " fwd (err / mag)", _tau_reached(y, y64, ymag, None, bf16=True), TAU)
    parity(name + " dgrad (err / mag)", _tau_reached(dx, dx64, dxmag, None, bf16=True), TAU)
    parity(name + " wgrad (err / mag)", _tau_reached(dw, dw64, dwmag, None, bf16=False), TAU_ACC)


# ------------------------------------------------------------------------------------------ (i) refusals
def test_host_refusals_leave_outputs_untouched():
    """Invalid calls are refused by host checks before any launch: the output keeps its sentinel."""
    from espresso_b200 import lib

    ops = _ops()
    M, N, K = 64, 64, 64
    a, b = _rand((M, K + 8), "randn", 1), _rand((N, K + 8), "randn", 2)
    c = _sentinel((M, N), F32)
    c16 = _sentinel((M, N), BF)
    aux = _rand((M, N), "randn", 3)
    bad = [
        ("16-byte aligned", lambda: ops.gemm(a.view(-1)[1:], b, c, M, N, K, K + 8, K + 8, N)),
        ("16-byte aligned", lambda: ops.gemm(a, b.view(-1)[3:], c, M, N, K, K + 8, K + 8, N)),
        ("multiple of 8", lambda: ops.gemm(a, b, c, M, N, K, K + 4, K + 8, N)),
        ("multiple of 8", lambda: ops.gemm(a, b, c, M, N, K, K + 8, K + 6, N)),
        ("batch strides", lambda: ops.gemm(a, b, c, 32, N, K, K + 8, K + 8, N, nb1=2, sA=(32 * (K + 8) + 4, 0),
                                           sC=(32 * N, 0))),
        ("bad GEMM shape", lambda: ops.gemm(a, b, c, M, N, 0, K + 8, K + 8, N)),
        ("must be fp32", lambda: ops.gemm(a, b, c16, M, N, K, K + 8, K + 8, N, accumulate=True)),
        ("needs aux", lambda: ops.gemm(a, b, c, M, N, K, K + 8, K + 8, N, act=ops.ACT_RELU_BWD)),
        ("needs aux", lambda: ops.gemm(a, b, c, M, N, K, K + 8, K + 8, N, act=ops.ACT_SILU_BWD)),
        ("rowsum_a", lambda: ops.gemm(a, b, c, M, N, K, K + 8, K + 8, N, accumulate=True,
                                      rowsum_a=torch.zeros(M, device="cuda"))),
        ("rowsum_a", lambda: ops.gemm(a, b, c, 32, N, K, K + 8, K + 8, N, a_kmajor=False, accumulate=True, nb1=2,
                                      sA=(32, 0), sC=(32 * N, 0), rowsum_a=torch.zeros(M, device="cuda"))),
    ]
    for msg, call in bad:
        with pytest.raises(lib.EspressoB200Error, match=msg):
            call()
    torch.cuda.synchronize()
    _assert_untouched(c, c[:0], "refused GEMM output")
    _assert_untouched(c16, c16[:0], "refused GEMM output")
    # empty shapes are no-ops
    ops.gemm(a, b, c, 0, N, K, K + 8, K + 8, N)
    ops.gemm(a, b, c, M, 0, K, K + 8, K + 8, N, bias=aux[0], act=ops.ACT_RELU_BWD, aux=aux, ld_aux=N)
    torch.cuda.synchronize()
    _assert_untouched(c, c[:0], "empty GEMM output")
    x = _rand((1, 8, 8, 32), "randn", 4)
    with pytest.raises(lib.EspressoB200Error, match="multiples of 64"):
        ops.conv3x3_fwd(x, _rand((64, 3, 3, 32), "randn", 5), (1, 1))
    x = _rand((1, 8, 8, 64), "randn", 6)
    with pytest.raises(lib.EspressoB200Error, match="strides 1 or 2"):
        ops.conv3x3_fwd(x, _rand((64, 3, 3, 64), "randn", 7), (3, 1))
    with pytest.raises(lib.EspressoB200Error, match="multiples of 64"):
        ops.conv3x3_dgrad(_rand((1, 8, 8, 96), "randn", 8), _rand((96, 3, 3, 64), "randn", 9), (1, 8, 8, 64), (1, 1))
    with pytest.raises(lib.EspressoB200Error, match="strides 1 or 2"):
        ops.conv3x3_wgrad(_rand((1, 8, 8, 64), "randn", 8), x, torch.zeros(64, 3, 3, 64, device="cuda"), (1, 3))
