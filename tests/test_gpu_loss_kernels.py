"""The three fused loss kernels (esp_ctc_loss, esp_rnnt_loss, esp_lsce_loss) against the float64 references of
oracle/loss64.py, on every branch of the kernels and at recipe shapes.  Each case names the branch it reaches.

Bounds, through the `parity` fixture (achieved errors are recorded next to them):
  loss       |L - L64| <= 1e-5 * max(1, |L64|)
  gradient   |g - g64| <= 2^-8 |g64| + a       2^-8 |g| bounds the bf16 rounding of the stored gradient; the floor `a`
                                               (per case, about 2x what an H100 reaches, at least FLOOR) covers the
                                               fp32 arithmetic
  row sums   |sum_v g| <= sum_v halfulp(g) + a_sum   every gradient row sums to 0 in exact arithmetic (softmax mass
                                               minus occupancy mass); the bf16 rounding of each stored value is at most
                                               half its ulp.  This catches missing occupancy mass (a dropped state or
                                               lattice cell) where the elementwise check is noisy.
Layout: the pad columns [V, ceil8(V)) are exactly 0, and a call through the C ABI into a sentinel-filled buffer writes
nothing outside the columns documented in include/espresso_b200.h.  The wrappers' gradients have the logits' strides.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import loss64

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
SENTINEL = -1024.0  # exactly representable in bf16; no gradient value comes near it
REL = 2.0 ** -8
# Floor of the cases where an H100 reaches 0 (or < 5e-7): a few fp32 ulps of an O(1) gradient value.  Twice zero is
# no bound; the cases with real fp32 error (long targets, large |loss|) carry their own floors, measured on an
# H100 SXM 80 GB at a 400 W power limit.
FLOOR = 1e-6


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


def _c8(v):
    return (v + 7) // 8 * 8


def _halfulp(g):
    """Half the bf16 ulp of each (bf16-representable) value of g; 0 for 0."""
    _, e = torch.frexp(g)
    return torch.where(g == 0, torch.zeros_like(g), torch.ldexp(torch.ones_like(g), e - 9))


def _check_loss(parity, name, loss, ref, bound=1e-5):
    err = ((loss.double() - ref).abs() / ref.abs().clamp(min=1.0)).max().item()
    parity("%s: loss |L-L64|/max(1,|L64|)" % name, err, bound)


def _check_grad(parity, name, g, ref, a, a_sum):
    """g: kernel gradient (bf16 values, any float dtype) [..., V]; ref: float64 [..., V]."""
    g = g.double()
    elem = ((g - ref).abs() - REL * ref.abs()).max().item()
    parity("%s: grad max(|g-g64| - 2^-8|g64|)" % name, max(elem, 0.0), a)
    rows = (g.sum(-1).abs() - _halfulp(g).sum(-1)).max().item()
    parity("%s: grad row sums max(|sum g| - sum halfulp(g))" % name, max(rows, 0.0), a_sum)


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _sentinel_like(x, extra=64):
    """(storage, view): a sentinel-filled buffer and a view of it with x's shape and strides, 16-byte aligned, with
    `extra` sentinel elements on both sides."""
    last = sum((n - 1) * s for n, s in zip(x.shape[:-1], x.stride()[:-1]))
    storage = torch.full((last + max(x.shape[-1], 8) + 8 + 2 * extra,), SENTINEL, dtype=BF, device=x.device)
    return storage, storage.as_strided(x.shape, x.stride(), extra)


def _check_layout(storage, view, rows_ld, V, gref, atol=None):
    """Positions of `storage` written by the kernel must be exactly the first rows_ld columns of every row of `view`
    (columns [V, rows_ld) equal to 0); everything else keeps the sentinel.  gref: the wrapper's gradient of the same
    call, which the written values equal exactly, or (atol given: the CTC occupancy sums use atomics, whose order
    varies) to one bf16 ulp + atol."""
    rows_shape = view.shape[:-1]
    base = view.storage_offset()
    offs = torch.zeros(rows_shape, dtype=torch.long, device=storage.device) + base
    for d, (n, s) in enumerate(zip(rows_shape, view.stride()[:-1])):
        shape = [1] * len(rows_shape)
        shape[d] = n
        offs = offs + (torch.arange(n, device=storage.device) * s).view(shape)
    cols = torch.arange(rows_ld, device=storage.device)
    written = (offs[..., None] + cols).reshape(-1)
    mask = torch.zeros(storage.numel(), dtype=torch.bool, device=storage.device)
    mask[written] = True
    assert (storage[~mask] == SENTINEL).all(), "kernel wrote outside the documented columns"
    w = storage[(offs[..., None] + cols)]
    assert (w[..., V:] == 0).all(), "pad columns not zeroed"
    gv, gr = w[..., :V].float(), gref[..., :V].float()
    if atol is None:
        assert torch.equal(gv, gr)
    else:
        assert ((gv - gr).abs() <= 2.0 ** -7 * gr.abs() + atol).all()


# ==================================================================================================================== CTC
def _ctc_ld_pad(B, T, sb, st, V):
    """Columns written per row (esp_ctc_loss comment in include/espresso_b200.h)."""
    if B == 1 and T > 1:
        m = st
    elif T == 1 and B > 1:
        m = sb
    else:
        m = min(sb, st)
    return _c8(V) if m >= _c8(V) else V


def _ctc_check(dev, parity, name, x, V, in_lens, tg, tl, blank, a, a_sum, zero_infinity=True, grad_scale=1.0,
               loss_bound=1e-5):
    """x: bf16 CUDA view [B, T, >=V].  Runs the wrapper and the C ABI into a sentinel buffer; checks both."""
    from espresso_b200 import lib, ops

    B, T, Cw = x.shape
    in_d, tg_d, tl_d = in_lens.to(dev), tg.to(dev), tl.to(dev)
    loss, grad = ops.ctc_loss(x, V, in_d, tg_d, tl_d, blank, zero_infinity=zero_infinity, grad_scale=grad_scale)
    assert grad.stride() == x.stride()
    L = lib.load()
    storage, gview = _sentinel_like(x)
    ws = torch.empty(int(L.esp_ctc_workspace_bytes(B, T, tg.shape[1])), device=dev, dtype=torch.uint8)
    loss2 = torch.empty(B, device=dev)
    lib.check(L.esp_ctc_loss(_ptr(x), x.stride(0), x.stride(1), V, B, T, _ptr(in_d), _ptr(tg_d.contiguous()), tg.shape[1],
                             _ptr(tl_d), blank, int(zero_infinity), float(grad_scale), _ptr(loss2), _ptr(gview), _ptr(ws),
                             _stream()))
    torch.cuda.synchronize()
    ld_pad = _ctc_ld_pad(B, T, x.stride(0), x.stride(1), V)
    _check_layout(storage, gview, ld_pad, V, grad, atol=2e-6 * grad_scale)
    assert torch.equal(loss, loss2)
    ref_l, ref_g = loss64.ctc(x.cpu(), V, in_lens, tg, tl, blank, zero_infinity=zero_infinity)
    ref_g = ref_g * grad_scale
    loss, g = loss.cpu(), grad.cpu()
    if Cw > V:
        assert not g[..., V:min(Cw, ld_pad)].any()
    fin = torch.isfinite(ref_l)
    assert torch.equal(torch.isfinite(loss), fin) and (loss[~fin] == float("inf")).all()
    _check_loss(parity, "ctc " + name, loss[fin], ref_l[fin], loss_bound)
    rows = []
    for b in range(B):
        # infeasible (reference loss inf, or 0 under zero_infinity): the kernel writes a zero gradient, which under
        # zero_infinity is the exact answer; otherwise rows t >= in_lens[b] are zero
        n = int(in_lens[b]) if bool(fin[b]) and ref_l[b] != 0 else 0
        assert not g[b, n:, :V].any(), (name, b)
        rows += [(b, t) for t in range(n)]
    if rows:
        bi, ti = torch.tensor(rows).t()
        _check_grad(parity, "ctc " + name, g[bi, ti, :V], ref_g[bi, ti], a, a_sum)
    return loss, g, ref_l, ref_g


def _rand_targets(rs, B, u_max, V, blank):
    labels = np.array([v for v in range(V) if v != blank])
    return torch.from_numpy(labels[rs.randint(0, len(labels), size=(B, max(u_max, 1)))].astype(np.int32))


def _ctc_logits(dev, rs, B, T, ld, scale=1.5):
    return torch.from_numpy((rs.randn(B, T, ld) * scale).astype(np.float32)).to(BF).to(dev)


def _min_frames(tg_row):
    t = list(tg_row)
    return len(t) + sum(1 for i in range(1, len(t)) if t[i] == t[i - 1])


# (a, a_sum): the occupancy exp(alpha + beta - lp + nll) is formed from fp32 terms of magnitude |nll| ~ 1e3 here, so
# its absolute error grows with the loss.  H100 reached (1.3e-4, 0), (6.3e-5, 0), (1.1e-3, 3.3e-4).
CTC_SCAN_FLOORS = {255: (3e-4, FLOOR), 256: (1.3e-4, FLOOR), 511: (2.2e-3, 7e-4)}


@pytest.mark.parametrize("u_max", [255, 256, 511])
def test_ctc_scan_states_per_thread(dev, parity, u_max):
    """u_max 255: one extended state per scan thread (C = 1); 256 and 511: the C = 2 instantiation, selected by the
    padded target width, so the short utterances of the batch run it too.  511 is the longest target supported."""
    a, a_sum = CTC_SCAN_FLOORS[u_max]
    rs = np.random.RandomState(u_max)
    V, B = 64, 4
    tl = torch.tensor([u_max, u_max - 37, 3, 0], dtype=torch.int32)
    tg = _rand_targets(rs, B, u_max, V, 0)
    T = int(u_max * 1.3) + 12
    in_lens = torch.tensor([T, T - 40, 9, 5], dtype=torch.int32)
    _ctc_check(dev, parity, "u_max=%d (scan C=%d)" % (u_max, 2 if u_max >= 256 else 1), _ctc_logits(dev, rs, B, T, V),
               V, in_lens, tg, tl, 0, a=a, a_sum=a_sum)


def test_ctc_target_too_long_is_an_error(dev):
    """u_max = 512 exceeds the register scan: the library raises before launching anything."""
    from espresso_b200 import lib, ops

    x = torch.zeros(1, 1200, 16, dtype=BF, device=dev)
    tg = torch.ones(1, 512, dtype=torch.int32, device=dev)
    n0 = lib.launch_count()
    with pytest.raises(lib.EspressoB200Error, match="u_max=512"):
        ops.ctc_loss(x, 16, torch.tensor([1200], dtype=torch.int32, device=dev), tg,
                     torch.tensor([512], dtype=torch.int32, device=dev), 0)
    torch.cuda.synchronize()
    assert lib.launch_count() == n0


@pytest.mark.parametrize("blank", ["last", "middle"])
def test_ctc_blank_not_zero(dev, parity, blank):
    """blank = V-1 and blank in the middle of the vocabulary (prep gathers and grad scatters at the blank index)."""
    rs = np.random.RandomState(11)
    V, B, T = 50, 3, 80
    bl = V - 1 if blank == "last" else 23
    tg = _rand_targets(rs, B, 25, V, bl)
    tl = torch.tensor([25, 17, 6], dtype=torch.int32)
    in_lens = torch.tensor([80, 61, 30], dtype=torch.int32)
    _ctc_check(dev, parity, "blank=%d" % bl, _ctc_logits(dev, rs, B, T, _c8(V)), V, in_lens, tg, tl, bl, a=FLOOR, a_sum=FLOOR)


def test_ctc_repeats_only(dev, parity):
    """Targets made only of repeats (no skip transition anywhere), one of them at its minimum length 2U - 1."""
    rs = np.random.RandomState(12)
    V, B, U = 30, 3, 20
    tg = torch.tensor([[7] * U, [3] * U, [29] * U], dtype=torch.int32)
    tl = torch.tensor([U, U, 9], dtype=torch.int32)
    in_lens = torch.tensor([2 * U - 1, 70, 40], dtype=torch.int32)
    _ctc_check(dev, parity, "repeats only", _ctc_logits(dev, rs, B, 70, 32), V, in_lens, tg, tl, 0, a=FLOOR, a_sum=FLOOR)


def test_ctc_single_alignment(dev, parity):
    """T' exactly at the feasibility minimum (U + #repeats): one alignment, so loss = -sum_t log p(path_t) and the
    gradient is softmax - onehot(path) exactly."""
    rs = np.random.RandomState(13)
    V, B = 40, 2
    tg = _rand_targets(rs, B, 60, V, 0)
    tg[:, 10:14] = 5  # three repeats
    tg[1, 30] = tg[1, 29]
    tl = torch.tensor([60, 45], dtype=torch.int32)
    T = [_min_frames(tg[b, : tl[b]].tolist()) for b in range(B)]
    in_lens = torch.tensor(T, dtype=torch.int32)
    x = _ctc_logits(dev, rs, B, max(T), 40)
    loss, g, ref_l, ref_g = _ctc_check(dev, parity, "single alignment", x, V, in_lens, tg, tl, 0, a=FLOOR, a_sum=FLOOR)
    # closed form, independent of any recursion
    lp = torch.log_softmax(x.cpu().double()[..., :V], -1)
    for b in range(B):
        path = []
        prev = None
        for y in tg[b, : tl[b]].tolist():
            if y == prev:
                path.append(0)
            path.append(y)
            prev = y
        assert len(path) == T[b]
        pt = torch.tensor(path)
        nll = -lp[b, torch.arange(T[b]), pt].sum()
        want = lp[b, : T[b]].exp()
        want[torch.arange(T[b]), pt] -= 1.0
        assert abs(ref_l[b] - nll) < 1e-9 * abs(nll) and (ref_g[b, : T[b]] - want).abs().max() < 1e-9
        _check_grad(parity, "ctc single alignment closed form, utt %d" % b, g[b, : T[b], :V], want, a=FLOOR, a_sum=FLOOR)


@pytest.mark.parametrize("zero_infinity", [True, False])
def test_ctc_infeasible_and_empty(dev, parity, zero_infinity):
    """T' one frame below the minimum (nll = inf), in_len = 0 with and without targets, next to feasible utterances
    that must be unaffected.  zero_infinity: loss 0 and zero gradient rows; otherwise loss inf (gradient rows 0)."""
    rs = np.random.RandomState(14)
    V, B, T = 20, 5, 50
    tg = _rand_targets(rs, B, 30, V, 0)
    tl = torch.tensor([30, 30, 10, 0, 12], dtype=torch.int32)
    in_lens = torch.tensor([50, _min_frames(tg[1, :30].tolist()) - 1, 0, 0, 45], dtype=torch.int32)
    loss, g, ref_l, _ = _ctc_check(dev, parity, "infeasible/in_len=0 zero_infinity=%d" % zero_infinity,
                                   _ctc_logits(dev, rs, B, T, 24), V, in_lens, tg, tl, 0, a=FLOOR, a_sum=FLOOR,
                                   zero_infinity=zero_infinity)
    assert loss[3] == 0  # no frames, no targets: the empty alignment
    if zero_infinity:
        assert loss[1] == 0 and loss[2] == 0
    else:
        assert loss[1] == float("inf") and loss[2] == float("inf")
    assert not g[1].any() and not g[2].any() and not g[3].any()
    assert torch.isfinite(loss[[0, 4]]).all() and g[0].any() and g[4].any()


@pytest.mark.parametrize("shape", ["B=1", "T=1", "B=1,T=1"])
def test_ctc_single_row_axes(dev, parity, shape):
    """The ld_pad special cases: with B == 1 only the time stride decides whether pad columns may be written, with
    t_max == 1 only the batch stride.  The other stride is set below ceil8(V) to show it is ignored."""
    rs = np.random.RandomState(15)
    V = 13
    B, T = {"B=1": (1, 40), "T=1": (3, 1), "B=1,T=1": (1, 1)}[shape]
    buf = _ctc_logits(dev, rs, max(B, T), 16, 1)
    strides = {"B=1": (1, 16, 1), "T=1": (16, 1, 1), "B=1,T=1": (16, 16, 1)}[shape]
    x = buf.as_strided((B, T, V), strides)
    tg = _rand_targets(rs, B, 6, V, 0)
    tl = torch.tensor([min(6, T)] * B, dtype=torch.int32)
    in_lens = torch.tensor([T] * B, dtype=torch.int32)
    _ctc_check(dev, parity, "single-row axis " + shape, x, V, in_lens, tg, tl, 0, a=FLOOR, a_sum=FLOOR)


@pytest.mark.parametrize("V", [9000, 10001])
def test_ctc_large_vocabulary(dev, parity, V):
    """V > 8192: the prep kernel's register cache overflows into the streaming loop; 10001 also has a scalar tail."""
    rs = np.random.RandomState(V)
    B, T = 2, 30
    tg = _rand_targets(rs, B, 10, V, 0)
    _ctc_check(dev, parity, "V=%d" % V, _ctc_logits(dev, rs, B, T, _c8(V)), V, torch.tensor([30, 21], dtype=torch.int32),
               tg, torch.tensor([10, 7], dtype=torch.int32), 0, a=FLOOR, a_sum=FLOOR)


@pytest.mark.parametrize("layout", ["ld=V=13", "misaligned base"])
def test_ctc_scalar_paths(dev, parity, layout):
    """Rows that are not 16-byte aligned: the scalar prep path (per row) and the scalar grad path."""
    rs = np.random.RandomState(16)
    B, T = 3, 30
    if layout == "ld=V=13":
        V = 13
        x = _ctc_logits(dev, rs, B, T, V)
    else:
        V = 100
        flat = _ctc_logits(dev, rs, 1, 1, B * T * 104 + 8).view(-1)
        x = flat[1:1 + B * T * 104].view(B, T, 104)
        assert x.data_ptr() % 16 == 2
    tg = _rand_targets(rs, B, 8, V, 0)
    _ctc_check(dev, parity, "scalar paths " + layout, x, V, torch.tensor([30, 25, 12], dtype=torch.int32), tg,
               torch.tensor([8, 8, 3], dtype=torch.int32), 0, a=FLOOR, a_sum=FLOOR)


@pytest.mark.parametrize("view", ["time slice", "column slice", "both"])
def test_ctc_strided_views(dev, parity, view):
    """Views of a larger buffer: the gradient must have the logits' strides, and its values sit at the strided
    positions (before the fix, the wrapper allocated a dense gradient that the kernel addressed with the view's
    strides)."""
    rs = np.random.RandomState(17)
    B, Tb, ldb = 3, 60, 1016
    buf = _ctc_logits(dev, rs, B, Tb, ldb)
    x = {"time slice": buf[:, :45], "column slice": buf[:, :, :1003], "both": buf[:, 5:50, :1003]}[view]
    V = 1003
    assert not x.is_contiguous()
    tg = _rand_targets(rs, B, 12, V, 0)
    _ctc_check(dev, parity, "strided view " + view, x, V, torch.tensor([45, 40, 20], dtype=torch.int32), tg,
               torch.tensor([12, 9, 4], dtype=torch.int32), 0, a=FLOOR, a_sum=FLOOR, grad_scale=0.5)


def _peaked_ctc(rs, B, T, V, tg, tl, in_lens, boost=15.0):
    """randn logits with one class per frame raised by `boost`: along a random alignment of the target on 90% of the
    frames, a random class elsewhere."""
    x = rs.randn(B, T, _c8(V)).astype(np.float32)
    for b in range(B):
        y = tg[b, : tl[b]].tolist()
        path = []
        for i, lab in enumerate(y):
            if i and lab == y[i - 1]:
                path.append(0)
            path.append(lab)
        n = int(in_lens[b])
        extra = n - len(path)
        ins = np.sort(rs.randint(0, len(path) + 1, size=extra))
        full, j = [], 0
        for i in range(len(path) + 1):
            while j < extra and ins[j] == i:
                full.append(0 if rs.rand() < 0.8 else path[min(i, len(path) - 1)])
                j += 1
            if i < len(path):
                full.append(path[i])
        for t in range(n):
            c = full[t] if rs.rand() < 0.9 else rs.randint(V)
            x[b, t, c] += boost
    return x


def test_ctc_long_peaked(dev, parity):
    """35 s of audio at 40 ms frames (T' = 875), V = 5004, U ~ 150, trained-like peaked logits: softmax - occupancy
    cancels, and the fp32 alpha / beta are large in magnitude."""
    rs = np.random.RandomState(18)
    V, B, T = 5004, 3, 875
    tg = _rand_targets(rs, B, 150, V, 0)
    tl = torch.tensor([150, 131, 40], dtype=torch.int32)
    in_lens = torch.tensor([875, 800, 300], dtype=torch.int32)
    x = torch.from_numpy(_peaked_ctc(rs, B, T, V, tg, tl, in_lens)).to(BF).to(dev)
    # H100 reached a = 1.7e-3, a_sum = 1.7e-3 (|nll| up to ~1e3: see CTC_SCAN_FLOORS)
    _ctc_check(dev, parity, "T'=875 V=5004 peaked", x, V, in_lens, tg, tl, 0, a=3.5e-3, a_sum=3.5e-3)


# ================================================================================================================= RNN-T
def _rnnt_check(dev, parity, name, x, V, t_lens, u_lens, tg, blank, a, a_sum, grad_scale=1.0, loss_bound=1e-5):
    from espresso_b200 import lib, ops

    B, T, U1, ld = x.shape
    tl_d, ul_d, tg_d = t_lens.to(dev), u_lens.to(dev), tg.to(dev)
    loss, grad = ops.rnnt_loss(x, V, tl_d, ul_d, tg_d, blank, grad_scale=grad_scale)
    assert grad.stride() == x.stride()
    L = lib.load()
    storage, gview = _sentinel_like(x)
    ws = torch.empty(int(L.esp_rnnt_workspace_bytes(B, T, U1)), device=dev, dtype=torch.uint8)
    loss2 = torch.empty(B, device=dev)
    lib.check(L.esp_rnnt_loss(_ptr(x), ld, V, B, T, U1, _ptr(tl_d), _ptr(ul_d), _ptr(tg_d), tg.shape[1], blank,
                              float(grad_scale), _ptr(loss2), _ptr(gview), _ptr(ws), _stream()))
    torch.cuda.synchronize()
    _check_layout(storage, gview, _c8(V), V, grad)
    loss, g = loss.cpu(), grad.cpu()
    assert torch.equal(loss, loss2.cpu())
    ref_l = torch.zeros(B, dtype=torch.float64)
    elems, refs = [], []
    for b in range(B):  # one utterance at a time keeps the float64 lattice small
        Tb, Ub = int(t_lens[b]), int(u_lens[b])
        lb, gb = loss64.rnnt(x[b:b + 1, :Tb, : Ub + 1].cpu(), V, t_lens[b:b + 1], u_lens[b:b + 1], tg[b:b + 1], blank)
        ref_l[b] = lb[0]
        elems.append(g[b, :Tb, : Ub + 1, :V].reshape(-1, V))
        refs.append(gb[0].reshape(-1, V) * grad_scale)
        assert not g[b, Tb:].any() and not g[b, :, Ub + 1:].any()
    _check_loss(parity, "rnnt " + name, loss, ref_l, loss_bound)
    _check_grad(parity, "rnnt " + name, torch.cat(elems), torch.cat(refs), a, a_sum)
    assert not g[..., V:_c8(V)].any()
    return loss, g


def _rnnt_logits(dev, g, B, T, U1, V, scale=1.5):
    x = torch.zeros(B, T, U1, _c8(V))
    x[..., :V] = torch.randn(B, T, U1, V, generator=g) * scale
    return x.to(BF).to(dev)


def _rnnt_targets(g, B, U, V, blank):
    labels = torch.tensor([v for v in range(V) if v != blank])
    return labels[torch.randint(0, len(labels), (B, max(U, 1)), generator=g)].int()


# gradient floor a: the arc posteriors exp(alpha + beta + lp - ll) come from fp32 terms of magnitude |ll| ~ 1e3 on these
# flat-logit lattices.  H100 reached 3.9e-6, 2.1e-5, 8.0e-5 (row sums 0).
RNNT_SCAN_FLOORS = {255: 8e-6, 256: 4.5e-5, 599: 1.6e-4}


@pytest.mark.parametrize("T,U,V", [(40, 255, 16), (30, 256, 16), (20, 599, 12)])
def test_rnnt_scan_u_stride(dev, parity, T, U, V):
    """U + 1 = 256 fills the 256-thread CTA; 257 and 600 make threads handle several u per anti-diagonal.
    U = 599 > T = 20."""
    g = torch.Generator().manual_seed(U)
    B = 2
    x = _rnnt_logits(dev, g, B, T, U + 1, V)
    _rnnt_check(dev, parity, "U+1=%d T=%d" % (U + 1, T), x, V, torch.tensor([T, T - 7], dtype=torch.int32),
                torch.tensor([U, U - 50], dtype=torch.int32), _rnnt_targets(g, B, U, V, 0), 0, a=RNNT_SCAN_FLOORS[U],
                a_sum=FLOOR)


@pytest.mark.parametrize("blank", ["last", "middle"])
def test_rnnt_blank_not_zero(dev, parity, blank):
    g = torch.Generator().manual_seed(21)
    V, B, T, U = 20, 3, 15, 8
    bl = V - 1 if blank == "last" else 9
    x = _rnnt_logits(dev, g, B, T, U + 1, V)
    _rnnt_check(dev, parity, "blank=%d" % bl, x, V, torch.tensor([15, 11, 6], dtype=torch.int32),
                torch.tensor([8, 5, 2], dtype=torch.int32), _rnnt_targets(g, B, U, V, bl), bl, a=FLOOR, a_sum=FLOOR)


def test_rnnt_small_vocabulary(dev, parity):
    """V = 5 < 8: the prep kernel has no vector loads, only its scalar loop."""
    g = torch.Generator().manual_seed(22)
    x = _rnnt_logits(dev, g, 2, 12, 7, 5)
    _rnnt_check(dev, parity, "V=5", x, 5, torch.tensor([12, 9], dtype=torch.int32), torch.tensor([6, 4], dtype=torch.int32),
                _rnnt_targets(g, 2, 6, 5, 0), 0, a=FLOOR, a_sum=FLOOR, grad_scale=0.25)


def test_rnnt_single_frame(dev, parity):
    """T = 1: the lattice is one row; every label is emitted at the first frame."""
    g = torch.Generator().manual_seed(23)
    x = _rnnt_logits(dev, g, 2, 1, 6, 24)
    _rnnt_check(dev, parity, "T=1", x, 24, torch.tensor([1, 1], dtype=torch.int32), torch.tensor([5, 2], dtype=torch.int32),
                _rnnt_targets(g, 2, 5, 24, 0), 0, a=FLOOR, a_sum=FLOOR)


def test_rnnt_ragged_with_empty_targets(dev, parity):
    """Ragged t_lens / u_lens in one batch, with U = 0 rows (a blank at every frame) and a one-frame utterance."""
    g = torch.Generator().manual_seed(24)
    V, B, T, U = 40, 4, 30, 10
    x = _rnnt_logits(dev, g, B, T, U + 1, V)
    _rnnt_check(dev, parity, "ragged with U=0 rows", x, V, torch.tensor([30, 12, 1, 20], dtype=torch.int32),
                torch.tensor([10, 0, 3, 0], dtype=torch.int32), _rnnt_targets(g, B, U, V, 0), 0, a=FLOOR, a_sum=FLOOR)


def test_rnnt_long_peaked(dev, parity):
    """T = 250, U = 100, V = 1000 with peaked logits: on a random monotone path every cell raises its next emission
    by 15; off the path each cell raises blank or a random class."""
    g = torch.Generator().manual_seed(25)
    V, B, T, U = 1000, 2, 250, 100
    t_lens = torch.tensor([250, 180], dtype=torch.int32)
    u_lens = torch.tensor([100, 70], dtype=torch.int32)
    tg = _rnnt_targets(g, B, U, V, 0)
    x = torch.zeros(B, T, U + 1, _c8(V))
    x[..., :V] = torch.randn(B, T, U + 1, V, generator=g)
    rnd = torch.randint(0, V, (B, T, U + 1), generator=g)
    off = torch.where(torch.rand(B, T, U + 1, generator=g) < 0.6, torch.zeros_like(rnd), rnd)
    x.scatter_add_(-1, off[..., None], torch.full((B, T, U + 1, 1), 15.0))
    for b in range(B):
        Tb, Ub = int(t_lens[b]), int(u_lens[b])
        moves = torch.cat([torch.zeros(Tb - 1), torch.ones(Ub)])[torch.randperm(Tb - 1 + Ub, generator=g)].tolist()
        t = u = 0
        for mv in moves + [0]:
            sym = int(tg[b, u]) if mv else 0
            x[b, t, u, sym] += 15.0
            x[b, t, u, int(off[b, t, u])] -= 15.0
            if mv:
                u += 1
            else:
                t += 1
    # H100 reached a = 7.0e-7, a_sum = 6.3e-7, and a loss error of 7.7e-6 of the 1e-5 bar, which is consistent with
    # ~1 fp32 ulp of the peaked logits (|x| ~ 16) in each of the T + U = 350 log-probs along the path.  The kernel is
    # deterministic, so the margin does not vary between runs.
    _rnnt_check(dev, parity, "T=250 U=100 V=1000 peaked", x.to(BF).to(dev), V, t_lens, u_lens, tg, 0, a=1.5e-6,
                a_sum=1.3e-6)


def test_rnnt_misaligned_base_is_an_error(dev):
    """The prep kernel reads rows as 16-byte vectors: a base that is not 16-byte aligned is refused before launch."""
    from espresso_b200 import lib, ops

    flat = torch.zeros(2 * 4 * 3 * 16 + 8, dtype=BF, device=dev)
    x = flat[1:1 + 2 * 4 * 3 * 16].view(2, 4, 3, 16)
    assert x.is_contiguous() and x.data_ptr() % 16 == 2
    n0 = lib.launch_count()
    with pytest.raises(lib.EspressoB200Error, match="aligned"):
        ops.rnnt_loss(x, 16, torch.tensor([4, 4], dtype=torch.int32, device=dev), torch.tensor([2, 2], dtype=torch.int32, device=dev),
                      torch.ones(2, 2, dtype=torch.int32, device=dev), 0)
    torch.cuda.synchronize()
    assert lib.launch_count() == n0


# ================================================================================================================= LS-CE
def _lsce_check(dev, parity, name, x, V, tg, pad, eps, smoothing, a, a_sum, unigram=None, U=0, grad_scale=1.0,
                chunk=4096):
    from espresso_b200 import lib, ops

    R = x.shape[0]
    tg_d = tg.to(dev)
    uni_d = None if unigram is None else unigram.to(dev)
    loss, nll, grad = ops.lsce_loss(x, V, tg_d, pad, eps, grad_scale=grad_scale, smoothing=smoothing, unigram=uni_d, U=U)
    assert grad.stride() == x.stride()
    storage, gview = _sentinel_like(x)
    loss2, nll2 = torch.empty(R, device=dev), torch.empty(R, device=dev)
    lib.check(lib.load().esp_lsce_loss(_ptr(x), x.stride(0), V, R, _ptr(tg_d), pad, eps, smoothing,
                                       None if uni_d is None else _ptr(uni_d), U, float(grad_scale), _ptr(loss2),
                                       _ptr(nll2), _ptr(gview), _stream()))
    torch.cuda.synchronize()
    _check_layout(storage, gview, _c8(V), V, grad)
    loss, nll = loss.cpu(), nll.cpu()
    assert torch.equal(loss, loss2.cpu()) and torch.equal(nll, nll2.cpu())
    xc, g = x.cpu(), grad.cpu()
    if x.shape[1] > V:
        assert not g[:, V:min(x.shape[1], _c8(V))].any()
    rl, rn = [], []
    worst = [0.0, 0.0]
    for r0 in range(0, R, chunk):  # float64 rows in slices keeps R = 26 000 x V = 5000 within host memory
        l64, n64, g64 = loss64.lsce(xc[r0:r0 + chunk], V, tg, pad, eps, smoothing, unigram, U, row0=r0)
        rl.append(l64)
        rn.append(n64)
        gc = g[r0:r0 + chunk, :V].double()
        g64 = g64 * grad_scale
        worst[0] = max(worst[0], ((gc - g64).abs() - REL * g64.abs()).max().item())
        worst[1] = max(worst[1], (gc.sum(-1).abs() - _halfulp(gc).sum(-1)).max().item())
    _check_loss(parity, "lsce " + name, loss, torch.cat(rl))
    _check_loss(parity, "lsce " + name + " (nll)", nll, torch.cat(rn))
    parity("lsce %s: grad max(|g-g64| - 2^-8|g64|)" % name, max(worst[0], 0.0), a)
    parity("lsce %s: grad row sums max(|sum g| - sum halfulp(g))" % name, max(worst[1], 0.0), a_sum)
    assert not g[tg == pad].any()
    return loss, nll, g


def _lsce_inputs(dev, rs, R, V, ld=None, pad=1, pad_frac=0.1, scale=2.0):
    ld = ld or _c8(V)
    x = torch.from_numpy((rs.randn(R, ld) * scale).astype(np.float32)).to(BF).to(dev)
    tg = rs.randint(0, V, size=R)
    tg[rs.rand(R) < pad_frac] = pad
    return x, torch.from_numpy(tg.astype(np.int32))


def _unigram(rs, V):
    u = rs.rand(V) ** 4 + 1e-3
    return torch.from_numpy((u / u.sum()).astype(np.float32))


@pytest.mark.parametrize("V", [2, 7, 8192, 8200, 32000])
@pytest.mark.parametrize("smoothing", [0, 1, 2])
def test_lsce_vocabulary_sizes(dev, parity, V, smoothing):
    """V = 2 and 7: scalar tail only (no vector loads); 8192: the register cache exactly full; 8200: one vector past
    it; 32000: mostly the streaming loop."""
    rs = np.random.RandomState(V + smoothing)
    U = 8
    x, tg = _lsce_inputs(dev, rs, 8 * U, V, pad=1 if V > 2 else 0)
    _lsce_check(dev, parity, "V=%d smoothing=%d" % (V, smoothing), x, V, tg, 1 if V > 2 else 0, 0.1, smoothing,
                a=FLOOR, a_sum=FLOOR, unigram=_unigram(rs, V) if smoothing == 1 else None, U=U)


@pytest.mark.parametrize("smoothing", [0, 1, 2])
def test_lsce_eps_zero_is_nll(dev, parity, smoothing):
    """eps = 0: every smoothing type reduces to the NLL, bit for bit."""
    rs = np.random.RandomState(30 + smoothing)
    V, U = 1000, 10
    x, tg = _lsce_inputs(dev, rs, 6 * U, V)
    loss, nll, g = _lsce_check(dev, parity, "eps=0 smoothing=%d" % smoothing, x, V, tg, 1, 0.0, smoothing, a=1e-2,
                               a_sum=1e-2, unigram=_unigram(rs, V) if smoothing == 1 else None, U=U)
    assert torch.equal(loss, nll)


def test_lsce_temporal_sentence_edges(dev, parity):
    """Temporal smoothing on right-padded sentences of lengths 1, 2, 3 and U: neighbours at +-1 / +-2 fall off the
    sentence or onto <pad> and carry no mass."""
    rs = np.random.RandomState(31)
    V, U, pad = 50, 9, 1
    x, _ = _lsce_inputs(dev, rs, 4 * U, V)
    tg = torch.from_numpy(rs.randint(2, V, size=(4, U)).astype(np.int32))
    for b, n in enumerate((1, 2, 3, U)):
        tg[b, n:] = pad
    _lsce_check(dev, parity, "temporal sentence edges", x, V, tg.view(-1), pad, 0.1, 2, a=FLOOR, a_sum=FLOOR, U=U)


@pytest.mark.parametrize("smoothing", [0, 2])
def test_lsce_many_rows(dev, parity, smoothing):
    """R = 26 000 target tokens (a large decoder batch), V = 5000."""
    rs = np.random.RandomState(32 + smoothing)
    V, U = 5000, 26
    x, tg = _lsce_inputs(dev, rs, 26000, V)
    _lsce_check(dev, parity, "R=26000 V=5000 smoothing=%d" % smoothing, x, V, tg, 1, 0.1, smoothing, a=FLOOR, a_sum=FLOOR,
                U=U)


@pytest.mark.parametrize("view", ["row slice", "column slice"])
def test_lsce_strided_views(dev, parity, view):
    """Row and column slices of a larger buffer: the gradient has the logits' strides and its values sit at the
    strided positions."""
    rs = np.random.RandomState(33)
    buf, _ = _lsce_inputs(dev, rs, 300, 1016, ld=1016)
    x = buf[100:164] if view == "row slice" else buf[:, :1003]
    V = 1003
    tg = torch.from_numpy(rs.randint(0, V, size=x.shape[0]).astype(np.int32))
    _lsce_check(dev, parity, "strided view " + view, x, V, tg, 1, 0.1, 0, a=FLOOR, a_sum=FLOOR, grad_scale=0.5)


def test_lsce_misaligned_is_an_error(dev):
    """Rows are read and written as 16-byte vectors: a base that is not 16-byte aligned is refused before launch."""
    from espresso_b200 import lib, ops

    flat = torch.zeros(4 * 16 + 8, dtype=BF, device=dev)
    x = flat[1:1 + 4 * 16].view(4, 16)
    n0 = lib.launch_count()
    with pytest.raises(lib.EspressoB200Error, match="aligned"):
        ops.lsce_loss(x, 16, torch.zeros(4, dtype=torch.int32, device=dev), 1, 0.1)
    torch.cuda.synchronize()
    assert lib.launch_count() == n0
