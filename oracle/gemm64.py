"""Float64 statement of the wgmma GEMM (espresso_b200/csrc/gemm_tcgen05.cu) and of its three implicit-GEMM 3x3 convolutions.

TEST INFRASTRUCTURE ONLY.  Every operand is taken at its exact bf16 value and widened to float64, so each product is
exact and each sum is a float64 sum: the result stands in for exact arithmetic when the kernels' fp32 results are
checked.  Besides the value, every function returns a per-element MAGNITUDE: the same computation over absolute values
(|A| |B|^T for a GEMM, its batched and convolution analogues), carried through the epilogue step by step.  A kernel that
accumulates and finishes in fp32 stays within  tau * magnitude  of the value for a tau of a few fp32 roundings of the
reduction; a single bf16 rounding anywhere on the way costs up to 2^-9 of the magnitude.

`gemm` has the signature of `espresso_b200.ops.gemm` and follows the kernel's epilogue order (epilogue32):
  v = acc + bias;  C2 <- bf16(v);  dropout mode 2;  activation (ReLU, SiLU, ReLU' with aux > 0, SiLU');  dropout mode 1;
  * alpha;  + beta * R (bf16, fp32, or the skewed BD[m, (skew_r - 1) - m + n]);  store.
With accumulate = True:  C += alpha * acc  and  rowsum_a += rowsum_scale * sum_k A.
Nothing is written: the returned tensors are logical [nb2, nb1, M, N] float64 (C_out, rowsum_a and the operands are only
read).  Runs on the device of its operands (cuBLAS DGEMM on a GPU) or on the CPU.
"""
import torch

from oracle import ops_ref as _ref

ACT_NONE, ACT_RELU, ACT_SILU, ACT_RELU_BWD, ACT_SILU_BWD = 0, 1, 2, 3, 4
F64 = torch.float64


class Result:
    """c, mag: value and magnitude of the output; apx: coefficient of the sigmoid approximation error (SiLU / SiLU'
    epilogues: the kernel's error grows by apx * max|sigmoid~ - sigmoid|); c2, mag2: the pre-activation side output;
    rowsum, rowsum_mag: the row sums of A (accumulate with rowsum_a)."""

    def __init__(self, **kw):
        self.c = self.mag = self.apx = self.c2 = self.mag2 = self.rowsum = self.rowsum_mag = None
        self.__dict__.update(kw)


def _view(t, nb2, nb1, rows, cols, s2, s1, ld, kmajor):
    stride = (s2, s1, ld, 1) if kmajor else (s2, s1, 1, ld)
    return t.as_strided((nb2, nb1, rows, cols), stride)


def _drop_mask(nb2, nb1, M, N, p, seed, dev):
    """Keep mask and fp32 rescale of the epilogue dropout at logical index (bt * M + m) * N + n, bt = b2 * nb1 + b1."""
    keep = _ref._keep(seed, _ref._flat_index(nb2, nb1, M, N), p).to(dev)
    return keep, _ref._dscale(p)


def gemm(A, B, C_out, M, N, K, lda, ldb, ldc, *, a_kmajor=True, b_kmajor=True, nb1=1, nb2=1, sA=(0, 0), sB=(0, 0),
         sC=(0, 0), bias=None, act=ACT_NONE, aux=None, ld_aux=0, sAux=(0, 0), R=None, ldr=0, sR=(0, 0), alpha=1.0,
         beta=1.0, C2=None, drop_p=0.0, drop_mode=0, seed=0, skew_r=0, tile_n=0, accumulate=False, rowsum_a=None,
         rowsum_scale=1.0):
    dev = A.device
    a = _view(A, nb2, nb1, M, K, sA[1], sA[0], lda, a_kmajor).to(F64)
    b = _view(B, nb2, nb1, N, K, sB[1], sB[0], ldb, b_kmajor).to(F64)
    v = a @ b.transpose(-1, -2)
    mag = a.abs() @ b.abs().transpose(-1, -2)
    out = Result()
    if accumulate:
        c0 = _view(C_out, nb2, nb1, M, N, sC[1], sC[0], ldc, True).to(F64)
        out.c = c0 + alpha * v
        out.mag = c0.abs() + abs(alpha) * mag
        out.apx = torch.zeros_like(mag)
        if rowsum_a is not None:
            r0 = rowsum_a[:M].to(F64)
            out.rowsum = r0 + rowsum_scale * a.sum(dim=(0, 1, 3))
            out.rowsum_mag = r0.abs() + abs(rowsum_scale) * a.abs().sum(dim=(0, 1, 3))
        return out
    if bias is not None:
        bv = bias[:N].to(F64)
        v = v + bv
        mag = mag + bv.abs()
    if C2 is not None:
        out.c2, out.mag2 = v.clone(), mag.clone()
    if drop_mode in (1, 2) and drop_p > 0:
        keep, dscale = _drop_mask(nb2, nb1, M, N, drop_p, seed, dev)
    if drop_mode == 2 and drop_p > 0:
        v = torch.where(keep, v * dscale, torch.zeros_like(v))
        mag = torch.where(keep, mag * dscale, torch.zeros_like(mag))
    apx = torch.zeros_like(v)
    if act == ACT_RELU:
        v = v.clamp_min(0)  # 1-Lipschitz: the magnitude carries over (a value within its error of 0 may land either side)
    elif act == ACT_SILU:
        s = torch.sigmoid(v)
        apx = v.abs()  # v * (sigmoid~(v) - sigmoid(v))
        v = v * s
        mag = 1.1 * mag  # |silu'| <= 1.0998
    elif act in (ACT_RELU_BWD, ACT_SILU_BWD):
        u = _view(aux, nb2, nb1, M, N, sAux[1], sAux[0], ld_aux, True).to(F64)
        if act == ACT_RELU_BWD:
            g = (u > 0).to(F64)  # strict: aux == 0 passes no gradient
            gmag = g
        else:
            s = torch.sigmoid(u)
            g = s * (1 + u * (1 - s))
            gmag = s * (1 + u.abs() * (1 - s))  # scale of the terms of g (g itself crosses 0 near u = -1.28)
            apx = v.abs() * (1 + u.abs())  # |dg / dsigmoid| <= 1 + |u|
        v = v * g
        mag = mag * gmag
    if drop_mode == 1 and drop_p > 0:
        v = torch.where(keep, v * dscale, torch.zeros_like(v))
        mag = torch.where(keep, mag * dscale, torch.zeros_like(mag))
        apx = torch.where(keep, apx * dscale, torch.zeros_like(apx))
    if alpha != 1.0:
        v, mag, apx = v * alpha, mag * abs(alpha), apx * abs(alpha)
    if R is not None:
        if skew_r:
            T = skew_r
            full = _view(R, nb2, nb1, M, 2 * T - 1, sR[1], sR[0], ldr, True).to(F64)
            i = torch.arange(M, device=dev)[:, None]
            j = torch.arange(N, device=dev)[None, :]
            r = full.gather(-1, ((T - 1) - i + j).expand(nb2, nb1, M, N))
        else:
            r = _view(R, nb2, nb1, M, N, sR[1], sR[0], ldr, True).to(F64)
        v = v + beta * r
        mag = mag + abs(beta) * r.abs()
    out.c, out.mag, out.apx = v, mag, apx
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 3x3 convolutions, zero padding 1, channels-last (espresso_b200/ops.py conv3x3_*): direct sums over the nine taps
# ---------------------------------------------------------------------------------------------------------------------
def _taps(T, F, st, sf):
    To, Fo = (T + st - 1) // st, (F + sf - 1) // sf
    for r in range(3):
        for s in range(3):
            # output (to, fo) reads input (to * st + r - 1, fo * sf + s - 1) = padded (to * st + r, fo * sf + s)
            yield r, s, slice(r, r + (To - 1) * st + 1, st), slice(s, s + (Fo - 1) * sf + 1, sf)


def _pad(x):
    return torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))


def conv3x3_fwd(x, w, stride):
    """y[b, to, fo, co] = sum_{r, s, ci} x[b, to*st + r - 1, fo*sf + s - 1, ci] w[co, r, s, ci] -> (y, magnitude)."""
    st, sf = stride
    B, T, F, Cin = x.shape
    xp, wd = _pad(x.to(F64)), w.to(F64)
    y = mag = 0
    for r, s, ti, fi in _taps(T, F, st, sf):
        xs = xp[:, ti, fi, :]
        y = y + torch.einsum("btfc,oc->btfo", xs, wd[:, r, s, :])
        mag = mag + torch.einsum("btfc,oc->btfo", xs.abs(), wd[:, r, s, :].abs())
    return y, mag


def conv3x3_dgrad(dy, w, in_shape, stride):
    """dx = the transpose of conv3x3_fwd applied to dy: each tap scatters dy . w[:, r, s, :] back to the input positions it
    read -> (dx [B, T, F, Cin], magnitude)."""
    st, sf = stride
    B, T, F, Cin = in_shape
    dyd, wd = dy.to(F64), w.to(F64)
    dxp = torch.zeros(B, T + 2, F + 2, Cin, dtype=F64, device=dy.device)
    magp = torch.zeros_like(dxp)
    for r, s, ti, fi in _taps(T, F, st, sf):
        dxp[:, ti, fi, :] += torch.einsum("btfo,oc->btfc", dyd, wd[:, r, s, :])
        magp[:, ti, fi, :] += torch.einsum("btfo,oc->btfc", dyd.abs(), wd[:, r, s, :].abs())
    return dxp[:, 1:T + 1, 1:F + 1, :], magp[:, 1:T + 1, 1:F + 1, :]


def conv3x3_wgrad(dy, x, stride, dw0=None):
    """dw[co, r, s, ci] = dw0 + sum_{b, to, fo} dy[b, to, fo, co] x[b, to*st + r - 1, fo*sf + s - 1, ci]
    -> (dw [Cout, 3, 3, Cin], magnitude)."""
    st, sf = stride
    B, T, F, Cin = x.shape
    Cout = dy.shape[-1]
    xp, dyd = _pad(x.to(F64)), dy.to(F64)
    dw = torch.zeros(Cout, 3, 3, Cin, dtype=F64, device=x.device)
    mag = torch.zeros_like(dw)
    for r, s, ti, fi in _taps(T, F, st, sf):
        xs = xp[:, ti, fi, :]
        dw[:, r, s, :] = torch.einsum("btfo,btfc->oc", dyd, xs)
        mag[:, r, s, :] = torch.einsum("btfo,btfc->oc", dyd.abs(), xs.abs())
    if dw0 is not None:
        dw, mag = dw + dw0.to(F64), mag + dw0.to(F64).abs()
    return dw, mag
