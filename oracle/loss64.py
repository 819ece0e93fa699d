"""Float64 references for the three fused loss kernels (csrc/ctc.cu, csrc/rnnt.cu, csrc/lsce.cu).

Each returns the per-utterance (or per-row) loss and the gradient of the summed loss w.r.t. the logits, both in
float64, from logits given in any float dtype.  They are the yardsticks of tests/test_gpu_loss_kernels.py and are
pinned by tests/test_loss_references.py.  Test infrastructure only.
"""
import numpy as np
import torch


# ---- CTC ------------------------------------------------------------------------------------------------------------
def ctc(logits, V, in_lens, targets, tgt_lens, blank, zero_infinity=True):
    """The reference criterion's own call in float64 (espresso/criterions/ctc_loss.py: log_softmax, then
    F.ctc_loss(reduction="none", zero_infinity)), differentiated by autograd.
    logits [B, T, >=V] -> (loss [B], grad [B, T, V]).  Rows t >= in_lens[b] get zero gradient."""
    x = logits[..., :V].detach().to("cpu", torch.float64).clone().requires_grad_(True)
    with torch.enable_grad():
        lp = torch.log_softmax(x, -1).transpose(0, 1)  # [T, B, V]
        tg = targets.long().cpu()
        if tg.dim() < 2 or tg.shape[1] == 0:
            tg = torch.zeros(x.shape[0], 1, dtype=torch.long)
        loss = torch.nn.functional.ctc_loss(lp, tg, in_lens.long().cpu(), tgt_lens.long().cpu(), blank=blank,
                                            reduction="none", zero_infinity=zero_infinity)
        loss.sum().backward()
    return loss.detach(), x.grad


# ---- RNN-T ----------------------------------------------------------------------------------------------------------
def _lattice(lpb, lpl):
    """log alpha, log beta over the [T, U+1] lattice by anti-diagonals (numpy float64).  lpb [T, U+1] blank log-probs,
    lpl [T, U] label log-probs.  alpha(t, u) = log P(reach (t, u)); beta(t, u) = log P(finish | at (t, u)), including
    the final blank.  Returns (alpha, beta, log-likelihood)."""
    T, U1 = lpb.shape
    ninf = -np.inf
    lpl = np.concatenate([lpl, np.full((T, 1), ninf)], axis=1)  # no label arc leaves the last column
    # one -inf guard row / column on each side, so that every neighbour index is in range
    alpha = np.full((T + 1, U1 + 1), ninf)  # alpha[t + 1, u + 1]
    beta = np.full((T + 1, U1 + 1), ninf)  # beta[t, u]
    for d in range(T + U1 - 1):
        u = np.arange(max(0, d - T + 1), min(d, U1 - 1) + 1)
        t = d - u
        a = np.logaddexp(alpha[t, u + 1] + lpb[t - 1, u], alpha[t + 1, u] + lpl[t, u - 1])  # from (t-1, u), (t, u-1)
        a[(t == 0) & (u == 0)] = 0.0
        alpha[t + 1, u + 1] = a
    beta[T - 1, U1 - 1] = lpb[T - 1, U1 - 1]
    for d in range(T + U1 - 3, -1, -1):
        u = np.arange(max(0, d - T + 1), min(d, U1 - 1) + 1)
        t = d - u
        beta[t, u] = np.logaddexp(beta[t + 1, u] + lpb[t, u], beta[t, u + 1] + lpl[t, u])  # to (t+1, u), (t, u+1)
    alpha, beta = alpha[1:, 1:], beta[:T, :U1]
    return alpha, beta, alpha[T - 1, U1 - 1] + lpb[T - 1, U1 - 1]


def rnnt(logits, V, t_lens, u_lens, targets, blank):
    """torchaudio.functional.rnnt_loss(fused_log_softmax=True, clamp=-1) restated in float64 with its analytic
    gradient.  logits [B, T, U1, >=V] -> (loss [B], grad [B, T, U1, V]); cells outside an utterance's lattice get
    zero gradient.  d(-ll)/dlogit_v at (t, u) = softmax_v * (gb + gl) - [v = blank] gb - [v = y_u] gl, where gb / gl
    are the posterior probabilities of the blank / label arc leaving (t, u)."""
    B, T, U1 = logits.shape[:3]
    loss = torch.zeros(B, dtype=torch.float64)
    grad = torch.zeros(B, T, U1, V, dtype=torch.float64)
    for b in range(B):
        Tb, Ub = int(t_lens[b]), int(u_lens[b])
        x = logits[b, :Tb, : Ub + 1, :V].detach().to("cpu", torch.float64).numpy()
        m = x.max(-1, keepdims=True)
        lse = m + np.log(np.exp(x - m).sum(-1, keepdims=True))
        lp = x - lse
        y = targets[b, :Ub].long().cpu().numpy()
        lpb = lp[:, :, blank]
        lpl = lp[:, np.arange(Ub), y] if Ub else np.zeros((Tb, 0))
        alpha, beta, ll = _lattice(lpb, lpl)
        loss[b] = -ll
        nb = np.full((Tb, Ub + 1), -np.inf)  # beta after the blank arc; finishing from (Tb-1, Ub) has probability 1
        nb[:-1] = beta[1:]
        nb[Tb - 1, Ub] = 0.0
        gb = np.exp(alpha + lpb + nb - ll)
        gl = np.zeros((Tb, Ub + 1))
        if Ub:
            gl[:, :Ub] = np.exp(alpha[:, :Ub] + lpl + beta[:, 1:] - ll)
        g = np.exp(lp) * (gb + gl)[..., None]
        g[:, :, blank] -= gb
        if Ub:
            tt, uu = np.meshgrid(np.arange(Tb), np.arange(Ub), indexing="ij")
            g[tt, uu, y[uu]] -= gl[:, :Ub]
        grad[b, :Tb, : Ub + 1] = torch.from_numpy(g)
    return loss, grad


def rnnt_autograd(logits, V, t_lens, u_lens, targets, blank):
    """Tiny lattices only: the plain float64 logsumexp recursion over every cell, differentiated by autograd.  It shares
    no formula with rnnt(), so it pins the analytic gradient there."""
    B = logits.shape[0]
    x = logits[..., :V].detach().to("cpu", torch.float64).clone().requires_grad_(True)
    losses = []
    with torch.enable_grad():
        lp = torch.log_softmax(x, -1)
        for b in range(B):
            Tb, Ub = int(t_lens[b]), int(u_lens[b])
            a = [[None] * (Ub + 1) for _ in range(Tb)]
            for t in range(Tb):
                for u in range(Ub + 1):
                    terms = []
                    if t == 0 and u == 0:
                        terms.append(torch.zeros((), dtype=torch.float64))
                    if t > 0:
                        terms.append(a[t - 1][u] + lp[b, t - 1, u, blank])
                    if u > 0:
                        terms.append(a[t][u - 1] + lp[b, t, u - 1, int(targets[b, u - 1])])
                    a[t][u] = torch.logsumexp(torch.stack(terms), 0)
            losses.append(-(a[Tb - 1][Ub] + lp[b, Tb - 1, Ub, blank]))
        loss = torch.stack(losses)
        loss.sum().backward()
    return loss.detach(), x.grad


# ---- label-smoothed cross-entropy -----------------------------------------------------------------------------------
UNIFORM, UNIGRAM, TEMPORAL = 0, 1, 2


def lsce(logits, V, targets, pad_idx, eps, smoothing=UNIFORM, unigram=None, U=0, row0=0):
    """espresso/criterions/label_smoothed_cross_entropy_v2.py in float64, for rows [row0, row0 + len(logits)) of a
    batch whose targets (all rows) are `targets`:
      uniform : loss = (1 - eps - eps/(V-1)) * nll + eps/(V-1) * sum_v -lp_v
      unigram : loss = (1 - eps) * nll + eps * sum_v u_v * -lp_v
      temporal: loss = (1 - eps) * nll + eps * sum_k m_k * -lp_{y_k}; rows are [B, U], y_k are the targets at distance
                -2, -1, +1, +2 inside the sentence with weights 2 : 5 : 5 : 2, <pad> neighbours dropped, normalised
    Rows whose target is <pad> give zero loss, nll and gradient.  With loss = a * nll + sum_v w_v * -lp_v the gradient is
    softmax * (a + sum w) - a * onehot(target) - w.  Returns (loss [n], nll [n], grad [n, V])."""
    x = logits[:, :V].detach().to("cpu", torch.float64).numpy()
    n = x.shape[0]
    tg_all = targets.long().cpu().numpy()
    r = np.arange(row0, row0 + n)
    tg = tg_all[r]
    m = x.max(-1, keepdims=True)
    lse = (m + np.log(np.exp(x - m).sum(-1, keepdims=True)))[:, 0]
    nll = lse - x[np.arange(n), tg]
    w = np.zeros((n, V))
    if smoothing == UNIFORM:
        a = 1.0 - eps - eps / (V - 1)
        w[:] = eps / (V - 1)
    elif smoothing == UNIGRAM:
        a = 1.0 - eps
        w[:] = eps * unigram[:V].detach().cpu().double().numpy()[None, :]
    else:
        a = 1.0 - eps
        pos = r % U
        tot = np.zeros(n)
        for off, c in ((-2, 2.0), (-1, 5.0), (1, 5.0), (2, 2.0)):
            ok = (pos + off >= 0) & (pos + off < U)
            nbr = np.where(ok, tg_all[np.clip(r + off, 0, len(tg_all) - 1)], pad_idx)
            ok &= nbr != pad_idx
            np.add.at(w, (np.arange(n)[ok], nbr[ok]), c)
            tot += np.where(ok, c, 0.0)
        w *= (eps / np.where(tot > 0, tot, 1.0))[:, None]
    sw = w.sum(-1)
    loss = a * nll + (w * (lse[:, None] - x)).sum(-1)
    g = np.exp(x - lse[:, None]) * (a + sw)[:, None] - w
    g[np.arange(n), tg] -= a
    keep = tg != pad_idx
    return (torch.from_numpy(np.where(keep, loss, 0.0)), torch.from_numpy(np.where(keep, nll, 0.0)),
            torch.from_numpy(g * keep[:, None]))
