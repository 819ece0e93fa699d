"""Pins the float64 loss references of oracle/loss64.py (the yardsticks of tests/test_gpu_loss_kernels.py) against
independent statements: oracle/ctc.py, torchaudio's rnnt_loss, autograd through a plain recursion, and the
label-smoothing outputs recorded from the reference implementation."""
import os

import numpy as np
import pytest
import torch

from oracle import ctc as octc
from oracle import loss64


def _ctc_case(seed, B, T, V, U, blank):
    rs = np.random.RandomState(seed)
    x = torch.from_numpy(rs.randn(B, T, V) * 2.0)
    labels = [v for v in range(V) if v != blank]
    tg = torch.from_numpy(rs.choice(labels, size=(B, max(U, 1)))).int()
    return x, tg


@pytest.mark.parametrize("blank", [0, 3, 6])
def test_ctc_reference_matches_oracle(blank):
    """Ragged lengths, repeated labels, a target at the feasibility minimum, an infeasible one, in_len = 0, U = 0."""
    V, T = 7, 9
    x, tg = _ctc_case(blank, 7, T, V, 5, blank)
    tg[2, 1] = tg[2, 0]  # one repeat: needs T >= U + 1
    tg[3] = tg[3, 0]  # only repeats: needs T >= 2U - 1 = 9
    in_lens = torch.tensor([9, 6, 6, 9, 3, 0, 0], dtype=torch.int32)
    tgt_lens = torch.tensor([5, 5, 5, 5, 5, 2, 0], dtype=torch.int32)  # row 4 is infeasible, row 5 has no frames
    for zi in (True, False):
        loss, grad = loss64.ctc(x, V, in_lens, tg, tgt_lens, blank, zero_infinity=zi)
        for b in range(x.shape[0]):
            nll, g = octc.ctc_loss_and_grad(x[b].numpy(), in_lens[b], tg[b, : tgt_lens[b]].numpy(), blank, zi)
            if np.isinf(nll):
                assert np.isinf(loss[b].item()) and not zi
                continue
            assert abs(loss[b].item() - nll) <= 1e-12 * max(1.0, abs(nll)), (b, zi)
            assert np.abs(grad[b].numpy() - g).max() <= 1e-12, (b, zi)
        assert loss[0] > 0 and loss[6] == 0  # U = 0 with no frames: the empty alignment
        if zi:
            assert loss[4] == 0 and loss[5] == 0 and not grad[4].any() and not grad[5].any()


def test_ctc_reference_single_alignment_closed_form():
    """T = U + #repeats admits one alignment: loss = -sum log p(path), gradient = softmax - onehot(path)."""
    V = 6
    x, _ = _ctc_case(5, 1, 6, V, 4, 0)
    tg = torch.tensor([[2, 2, 5, 1]], dtype=torch.int32)
    path = [2, 0, 2, 5, 1]
    x = x[:, :5]
    loss, grad = loss64.ctc(x, V, torch.tensor([5], dtype=torch.int32), tg, torch.tensor([4], dtype=torch.int32), 0)
    lp = torch.log_softmax(x[0], -1)
    assert abs(loss[0].item() + sum(lp[t, p].item() for t, p in enumerate(path))) < 1e-12
    want = lp.exp()
    want[torch.arange(5), torch.tensor(path)] -= 1.0
    assert (grad[0] - want).abs().max().item() < 1e-12


def _rnnt_case(seed, B, T, U, V, blank):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, U + 1, V, generator=g, dtype=torch.float64) * 1.5
    labels = torch.tensor([v for v in range(V) if v != blank])
    tg = labels[torch.randint(0, len(labels), (B, max(U, 1)), generator=g)].int()
    return x, tg


@pytest.mark.parametrize("B,T,U,V,blank", [(3, 7, 4, 6, 0), (2, 3, 6, 5, 4), (2, 5, 3, 9, 4), (2, 1, 3, 5, 2)])
def test_rnnt_reference_matches_torchaudio(B, T, U, V, blank):
    torchaudio = pytest.importorskip("torchaudio")
    x, tg = _rnnt_case(T * 7 + U, B, T, U, V, blank)
    t_lens = torch.tensor([T] + [max(1, T - i) for i in range(1, B)], dtype=torch.int32)
    u_lens = torch.tensor([U] + [max(0, U - 2 * i) for i in range(1, B)], dtype=torch.int32)
    loss, grad = loss64.rnnt(x, V, t_lens, u_lens, tg, blank)
    xf = x.float().clone().requires_grad_(True)
    ta = torchaudio.functional.rnnt_loss(xf, tg, t_lens, u_lens, blank=blank, clamp=-1.0, reduction="none")
    ta.sum().backward()
    assert ((loss - ta.detach().double()).abs() <= 1e-5 * loss.abs().clamp(min=1.0)).all(), (loss, ta)
    assert (grad - xf.grad.double()).abs().max().item() < 1e-5


@pytest.mark.parametrize("B,T,U,V,blank", [(2, 4, 3, 5, 0), (2, 3, 4, 6, 5), (1, 1, 2, 4, 1), (2, 5, 0, 4, 2)])
def test_rnnt_reference_matches_float64_autograd(B, T, U, V, blank):
    x, tg = _rnnt_case(100 + T + U, B, T, U, V, blank)
    t_lens = torch.tensor([T] + [max(1, T - 1)] * (B - 1), dtype=torch.int32)
    u_lens = torch.tensor([U] + [max(0, U - 1)] * (B - 1), dtype=torch.int32)
    loss, grad = loss64.rnnt(x, V, t_lens, u_lens, tg, blank)
    la, ga = loss64.rnnt_autograd(x, V, t_lens, u_lens, tg, blank)
    assert (loss - la).abs().max().item() < 1e-12
    assert (grad - ga).abs().max().item() < 1e-12
    # every cell's gradient row sums to zero, and outside the lattice it is zero
    assert grad.sum(-1).abs().max().item() < 1e-12
    for b in range(B):
        assert not grad[b, t_lens[b]:].any() and not grad[b, :, u_lens[b] + 1:].any()


def test_lsce_reference_matches_reference_fixture(golden_dir):
    """Uniform, unigram and temporal smoothing vs the reference's label_smoothed_nll_loss (+ its temporal mask) on the
    recorded fp32 logits; the fixture is fp32, so the agreement is at fp32 precision."""
    g = np.load(os.path.join(golden_dir, "label_smoothing.npz"))
    B, U, V = g["logits"].shape
    x = torch.from_numpy(g["logits"]).view(-1, V)
    tgt = torch.from_numpy(g["target"]).view(-1)
    pad = int(g["pad"])
    assert (tgt == pad).any()  # the fixture has right-padded sentences
    for name, mode in (("uniform", 0), ("unigram", 1), ("temporal", 2)):
        loss, nll, grad = loss64.lsce(x, V, tgt, pad, float(g["eps"]), mode, torch.from_numpy(g["unigram"]), U)
        assert abs(loss.sum().item() - float(g["loss_" + name])) < 2e-6 * abs(float(g["loss_" + name])), name
        assert abs(nll.sum().item() - float(g["nll_" + name])) < 2e-6 * abs(float(g["nll_" + name])), name
        assert np.abs(grad.numpy().reshape(B, U, V) - g["grad_" + name]).max() < 1e-6, name


def test_lsce_reference_row_slices_and_eps0():
    """Computing rows in slices (how the large GPU cases use it) gives the same answer, and eps = 0 is the NLL."""
    from oracle import ops_ref

    rs = np.random.RandomState(3)
    Bs, U, V, pad = 4, 6, 11, 1
    x = torch.from_numpy(rs.randn(Bs * U, V))
    tgt = torch.from_numpy(rs.randint(2, V, size=(Bs, U))).int()
    for b, n in enumerate((1, 2, 3, U)):
        tgt[b, n:] = pad
    tgt = tgt.view(-1)
    full = loss64.lsce(x, V, tgt, pad, 0.1, loss64.TEMPORAL, U=U)
    parts = [loss64.lsce(x[r:r + 5], V, tgt, pad, 0.1, loss64.TEMPORAL, U=U, row0=r) for r in range(0, Bs * U, 5)]
    for i in range(3):
        assert torch.equal(full[i], torch.cat([p[i] for p in parts]))
    # the bf16 oracle of ops_ref (dense weights) agrees on the same bf16-representable logits
    xb = x.bfloat16()
    lo, no, go = ops_ref.lsce_loss(xb, V, tgt, pad, 0.1, smoothing=2, U=U)
    l64, n64, g64 = loss64.lsce(xb, V, tgt, pad, 0.1, loss64.TEMPORAL, U=U)
    assert (lo.double() - l64).abs().max() < 1e-5 and (go.double() - g64).abs().max() < 4e-3
    for mode in (loss64.UNIFORM, loss64.TEMPORAL):
        loss, nll, grad = loss64.lsce(x, V, tgt, pad, 0.0, mode, U=U)
        assert torch.equal(loss, nll)
