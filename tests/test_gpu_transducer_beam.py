"""GPU: the transducer beam kernels (csrc/transducer_beam.cu) against their statements in oracle/transducer_beam_ops.py, and the
decoder's batched device search end to end."""
import copy
import os
import sys

import numpy as np
import pytest
import torch

from oracle import transducer_beam_ops as ops_ref

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")


def _state(B, K, beam, E, alpha, seed, nframes=None):
    """A search state with random rows and a random prefix pool (host copy, CPU)."""
    from espresso_b200.tools.transducer_beam_search_decoder import beam_state

    g = torch.Generator().manual_seed(seed)
    st = beam_state(B, K, beam, E, alpha, 64, torch.full((B,), 5, dtype=torch.int32) if nframes is None else nframes,
                    torch.device("cpu"))
    st["nrow"][:] = beam
    for b in range(B):
        for s in range(beam):
            node = 0
            for _ in range(int(torch.randint(0, 4, (1,), generator=g))):
                node = ops_ref._push_node(st, b, node, int(torch.randint(3, 9, (1,), generator=g)))
            r = b * K + s
            st["node"][r], st["len"][r] = node, int(st["p_len"][b * st["P"] + node])
            st["score"][r] = -float(torch.rand(1, generator=g)) * 5
            st["nemit"][r] = int(torch.randint(1, 6, (1,), generator=g))
    return st


def _to(st, dev):
    return {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in st.items() if k != "_struct"}


def _same_state(a, b, keys):
    for k in keys:
        x, y = a[k].cpu(), b[k].cpu()
        if x.dtype == torch.float32:
            assert torch.allclose(x, y, atol=1e-5, rtol=0, equal_nan=True), (k, x, y)
        else:
            assert torch.equal(x, y), (k, x, y)


@pytest.mark.parametrize("V,blank,pad,k,lm,nbl,fold,temp", [
    (5004, 0, 1, 7, False, False, False, 1.3), (5004, 4, 1, 7, True, True, False, 1.0), (50, 0, 1, 49, False, False, True, 1.0),
    (50, 0, 0, 50, True, False, True, 0.7), (37, 2, 1, 5, True, False, False, 1.0)])
def test_lprobs_matches_statement(V, blank, pad, k, lm, nbl, fold, temp):
    """V = 5004 and toy vocabularies; pad != blank (k clipped at V - 1) and pad == blank (k = V); LM fusion with and
    without blank in the LM's vocabulary; eos folding; equal logits and -inf scores (ties by token)."""
    from espresso_b200 import ops

    torch.manual_seed(V + k)
    n = 12
    ld = (V + 7) // 8 * 8
    logits = (torch.randn(n, ld) * 3).bfloat16()
    logits[3] = 0.5  # a row of equal logits
    scores = -torch.rand(n) * 4
    scores[5] = float("-inf")
    lml = torch.randn(n, V - int(nbl)) * 2 if lm else None
    args = (V, scores, k, blank, temp, 2, fold)
    kw = dict(lm_logits=lml, lm_weight=0.4, no_blank_in_lm=nbl) if lm else {}
    want = ops_ref.rnnt_beam_lprobs(logits, *args, **kw)
    if lm:
        kw["lm_logits"] = lml.to(DEV)
    got = ops.rnnt_beam_lprobs(logits.to(DEV), V, scores.to(DEV), *args[2:], **kw)
    torch.cuda.synchronize()
    assert torch.equal(got[1].cpu(), want[1])
    fin = torch.isfinite(want[0])
    assert torch.equal(torch.isfinite(got[0].cpu()), fin)
    assert (got[0].cpu()[fin] - want[0][fin]).abs().max() < 1e-5 * max(1.0, float(want[0][fin].abs().max()))
    assert (got[2].cpu() - want[2]).abs().max() < 1e-5


@pytest.mark.parametrize("alpha", [1, 2, 3])
def test_prefix_merge_and_scores_match_statement(alpha):
    """Random pools with chains that differ only at their first token, two different nodes spelling the same sequence,
    utterances outside their frames; merge pairs, ring rows and tokens exact, merged scores to 1e-5 (with and without
    an LM)."""
    from espresso_b200 import ops

    B, K, beam, E, V = 6, 7, 5, 3, 40
    st = _state(B, K, beam, E, alpha, alpha, nframes=torch.tensor([5, 5, 0, 5, 5, 5], dtype=torch.int32))
    # utterance 0: rows "a", "a b" (two nodes for "a b"), "c b": a prefix pair through a duplicate node, and a chain that
    # differs from "a b" only at its first token
    b, P = 0, st["P"]
    st["npool"][b] = 1
    n_a = ops_ref._push_node(st, b, 0, 5)
    n_ab = ops_ref._push_node(st, b, n_a, 6)
    n_a2 = ops_ref._push_node(st, b, 0, 5)
    n_ab2 = ops_ref._push_node(st, b, n_a2, 6)
    n_cb = ops_ref._push_node(st, b, ops_ref._push_node(st, b, 0, 7), 6)
    n_abx = ops_ref._push_node(st, b, n_ab2, 8)
    for s, nd in enumerate([n_a, n_ab, n_ab2, n_cb, n_abx]):
        st["node"][s], st["len"][s] = nd, int(st["p_len"][b * P + nd])
    assert int(st["p_hash"][n_ab]) == int(st["p_hash"][n_ab2])
    gpu = _to(st, DEV)
    ops_ref.rnnt_beam_prefix_merge(st, 1, alpha)
    ops.rnnt_beam_prefix_merge(gpu, 1, alpha)
    torch.cuda.synchronize()
    _same_state(gpu, st, ("score", "nemit", "len", "node", "srow", "fsrc", "nlive", "na", "m_npair"))
    assert int(st["m_npair"][0]) >= 3
    for b in range(B):
        n = int(st["m_npair"][b])
        Pm = st["Pm"]
        assert torch.equal(gpu["m_pair"][b * Pm * 4: b * Pm * 4 + 4 * n].cpu(), st["m_pair"][b * Pm * 4: b * Pm * 4 + 4 * n])
        last = st["m_pair"][b * Pm * 4 + 4 * n - 4: b * Pm * 4 + 4 * n] if n else None
        if n:
            hi = int(last[2] + last[3])
            assert torch.equal(gpu["m_ring"][b * st["S"]: hi].cpu(), st["m_ring"][b * st["S"]: hi])
            assert torch.equal(gpu["m_tok"][b * st["S"]: hi].cpu(), st["m_tok"][b * st["S"]: hi])
    for lm in (False, True):
        a, g = copy.deepcopy({k: v for k, v in st.items()}), _to(st, DEV)
        torch.manual_seed(alpha + 10 * lm)
        logits = (torch.randn(B * st["S"], 40) * 2).bfloat16()
        lml = torch.randn(B * st["S"], V - 1) if lm else None
        kw = dict(lm_logits=lml, lm_weight=0.4, no_blank_in_lm=True) if lm else {}
        ops_ref.rnnt_beam_merge_scores(logits, V, a, 1.3, 0, **kw)
        if lm:
            kw["lm_logits"] = lml.to(DEV)
        ops.rnnt_beam_merge_scores(logits.to(DEV), V, g, 1.3, 0, **kw)
        torch.cuda.synchronize()
        _same_state(g, a, ("score",))


@pytest.mark.parametrize("case", ["normal", "ties", "all_blank", "final", "nemit0", "done"])
def test_select_matches_statement(case):
    """One round (pruning, ranking, set-aside, pool growth, early combination), the final combination, equal scores,
    an all-blank round, nemit = 0 and an utterance that is done."""
    from espresso_b200 import ops

    B, K, beam, E = 5, 7, 5, 3
    k = 1 if case in ("all_blank", "nemit0") else K
    beam = 1 if k == 1 else beam
    st = _state(B, k if k == 1 else K, beam, E, 1, 7)
    K = st["K"]
    ops_ref.rnnt_beam_prefix_merge(st, 0, 1)
    if case == "done":
        st["nlive"][2] = 0
    if case == "nemit0":
        st["nemit"][:] = 0
    torch.manual_seed(3)
    val = torch.sort(-torch.rand(B * K, k) * 6, dim=1, descending=True)[0]
    tok = torch.stack([torch.randperm(12)[:k] for _ in range(B * K)]).int()
    if case == "ties":
        val[:, :] = -2.0
    if case in ("all_blank", "nemit0"):
        tok[:] = 0
        if case == "all_blank":
            tok[K] = 3  # utterance 1 has a non-blank proposal, the others do not
    lpb = -torch.rand(B * K)
    # one earlier round's set-aside entries
    for b in range(B):
        for q in range(2):
            a = b * st["A"] + q
            st["a_score"][a], st["a_nemit"][a], st["a_len"][a], st["a_src"][a] = -1.5 - q, 2, 1, b * K + q
        st["na"][b] = 2
    gpu = _to(st, DEV)
    final = case == "final"
    ops_ref.rnnt_beam_select(val, tok, lpb, st, 1, beam, 0, 2.3 if case != "ties" else None, True, final)
    ops.rnnt_beam_select(val.to(DEV), tok.to(DEV), lpb.to(DEV), gpu, 1, beam, 0, 2.3 if case != "ties" else None, True, final)
    torch.cuda.synchronize()
    _same_state(gpu, st, ("score", "nemit", "len", "node", "fsrc", "parent", "prev", "nrow", "nlive", "na", "npool", "a_score",
                          "a_nemit", "a_len", "a_node", "a_src", "p_parent", "p_tok", "p_len", "p_hash"))


def test_finalize_matches_statement():
    from espresso_b200 import ops

    st = _state(4, 7, 5, 2, 1, 11)
    st["nrow"][1] = 2
    st["score"][3] = st["score"][4]  # equal scores
    gpu = _to(st, DEV)
    want = ops_ref.rnnt_beam_finalize(st, 1)
    got = ops.rnnt_beam_finalize(gpu, 1)
    assert torch.equal(got[0].cpu(), want[0]) and torch.equal(got[2].cpu(), want[2])
    assert torch.allclose(got[1].cpu(), want[1], atol=1e-6, rtol=0)


class _D:
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def pad(self):
        return 1

    def eos(self):
        return 2

    def bos(self):
        return 0


def test_whole_fixture_batch_gives_reference_nbest(golden_dir):
    """All three fixture utterances in one call through the device path: every utterance's n-best has the reference's
    best tokens and scores within bf16 tolerance (the expectations of the host search's GPU test)."""
    from test_host_orchestration import _BEAM_CASES, _build_transducer, _lm_from_fixture
    from espresso_b200.tools.transducer_beam_search_decoder import TransducerBeamSearchDecoder

    g = np.load(os.path.join(golden_dir, "transducer_conformer.npz"))
    gg = np.load(os.path.join(golden_dir, "transducer_greedy.npz"))
    m = _build_transducer(g).finalize_(DEV)
    sample = {"net_input": {"src_tokens": torch.from_numpy(g["feats"]).to(DEV), "src_lengths": torch.from_numpy(g["lens"]).to(DEV)}}
    for name, kw, use_lm in _BEAM_CASES:
        if kw["prefix_alpha"] is None:
            continue
        lm = _lm_from_fixture(gg).finalize_(DEV, torch.float32) if use_lm else None
        dec = TransducerBeamSearchDecoder([m], _D(50), blank=0, lm_model=lm, lm_weight=0.3, **kw)
        hyps = dec.generate([m], sample)
        for b in range(3):
            ref_seqs, ref_scores = gg["%s_b%d_seqs" % (name, b)], gg["%s_b%d_scores" % (name, b)]
            assert abs(float(hyps[b][0]["score"]) - float(ref_scores[0])) < 0.05 * abs(float(ref_scores[0])) + 0.02
            if len(ref_scores) > 1 and ref_scores[0] - ref_scores[1] > 0.1:
                assert hyps[b][0]["tokens"].tolist() == [t for t in ref_seqs[0].tolist() if t != 1], (name, b)


def test_batch_invariance_on_a_random_model(golden_dir):
    """On the same encoder frames, each utterance decodes to the same n-best alone and inside a batch of utterances that
    end at different frames."""
    from test_host_orchestration import _build_transducer
    from espresso_b200.tools.transducer_beam_search_decoder import TransducerBeamSearchDecoder

    g = np.load(os.path.join(golden_dir, "transducer_conformer.npz"))
    m = _build_transducer(g).finalize_(DEV)
    torch.manual_seed(0)
    B, T, J = 4, 40, m.fc_out_weight()[0].shape[1]
    pe = (torch.randn(B, T, J, device=DEV) * 0.7).bfloat16()
    W = m.fc_out_weight()[0]
    lens = [40, 17, 29, 3]
    kw = dict(beam_size=5, max_num_expansions_per_step=4, expansion_beta=2, expansion_gamma=2.3, prefix_alpha=2, temperature=1.3)
    dec = TransducerBeamSearchDecoder([m], _D(50), blank=0, **kw)
    with torch.no_grad():
        both = dec._generate_batched(m, pe, W, lens, T, DEV, None)
        for b in range(B):
            alone = dec._generate_batched(m, pe[b:b + 1].contiguous(), W, lens[b:b + 1], T, DEV, None)
            assert torch.equal(alone[0][0].cpu(), both[b][0].cpu()), b
            assert torch.allclose(alone[0][1].cpu(), both[b][1].cpu(), atol=1e-5, rtol=0), b


def test_device_path_matches_host_search(golden_dir, monkeypatch):
    """The same decoder through the batched device search and through the per-utterance host search gives identical
    n-best tokens and scores within bf16 noise, with and without the LM."""
    from test_host_orchestration import _BEAM_CASES, _build_transducer, _lm_from_fixture
    from espresso_b200.tools.transducer_beam_search_decoder import TransducerBeamSearchDecoder

    g = np.load(os.path.join(golden_dir, "transducer_conformer.npz"))
    gg = np.load(os.path.join(golden_dir, "transducer_greedy.npz"))
    m = _build_transducer(g).finalize_(DEV)
    sample = {"net_input": {"src_tokens": torch.from_numpy(g["feats"]).to(DEV), "src_lengths": torch.from_numpy(g["lens"]).to(DEV)}}
    for name, kw, use_lm in _BEAM_CASES[:2]:
        lm = _lm_from_fixture(gg).finalize_(DEV, torch.float32) if use_lm else None
        dec = TransducerBeamSearchDecoder([m], _D(50), blank=0, lm_model=lm, lm_weight=0.3, **kw)
        dev_hyps = dec.generate([m], sample)
        monkeypatch.setattr(dec, "_generate_batched", dec._generate_host)
        host_hyps = dec.generate([m], sample)
        for b in range(3):
            assert [h["tokens"].tolist() for h in dev_hyps[b]] == [h["tokens"].tolist() for h in host_hyps[b]], (name, b)
            assert np.allclose([float(h["score"]) for h in dev_hyps[b]], [float(h["score"]) for h in host_hyps[b]], atol=1e-3)
