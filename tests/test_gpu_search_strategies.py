"""GPU: the search-option kernels (esp_beam_block_ngrams, esp_beam_prefix, esp_beam_diverse_groups, esp_beam_sibling_topk,
esp_beam_sample) against their per-op statements (sampled tokens bit for bit for the same seed, and a chi-square test of the
draws) in oracle/search_strategies.py on every branch, the generator end to end against the real
reference's hypotheses (tests/golden/search_strategies.npz), CUDA-graph replay against eager runs with a real model, and
the launches per search step of each option."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

DEV = torch.device("cuda:0")
NEG = float("-inf")


def test_block_ngrams_vs_statement():
    from espresso_b200 import ops
    from oracle import search_strategies as OS

    rs = np.random.RandomState(0)
    for V, alphabet in ((5004, 4), (5004, 5004), (9, 3)):
        for n in (1, 2, 3, 4):
            for step in (0, 1, n - 2, n - 1, n, 7, 40):
                if step < 0:
                    continue
                N, L = 6, 44  # the generator's full-width token buffer: columns after `step` hold stale values
                tok = torch.from_numpy(rs.randint(0, alphabet, size=(N, L))).int()
                tok[:, 0] = 2
                lp = torch.from_numpy(rs.randn(N, V).astype(np.float32))
                lp[1, :] = NEG
                lp[1, 7] = -0.5  # a row that is -inf except one token
                got = lp.to(DEV)
                ops.beam_block_ngrams(tok.to(DEV), step, n, got, V)
                want = OS.beam_block_ngrams(tok, step, n, lp.clone(), V)
                assert torch.equal(got.cpu(), want), (V, n, step)
                if step >= n - 1 and alphabet == 3:
                    assert torch.isinf(want).sum() > 0  # the case bans something


def test_prefix_vs_statement():
    from espresso_b200 import ops
    from oracle import search_strategies as OS

    class St:
        pass

    rs = np.random.RandomState(1)
    PAD, EOS = 1, 2
    for V, beam, bsz in ((5004, 5, 4), (11, 3, 4), (7, 1, 3)):
        N, L = bsz * beam, 12
        prefix = torch.tensor([[5, EOS, 6], [PAD, 4, PAD], [EOS, 3, 3], [6, 6, 6]][:bsz], dtype=torch.int32)
        for step in range(3):
            cand = torch.from_numpy(rs.randn(N, V).astype(np.float32))
            cand[0, 5] = NEG  # a forced token that is already -inf
            g, r = St(), St()
            g.tokens = torch.from_numpy(rs.randint(0, V, size=(N, L))).int()
            g.scores = torch.from_numpy(rs.randn(N, L - 1).astype(np.float32))
            r.tokens, r.scores = g.tokens.clone(), g.scores.clone()
            g.tokens, g.scores = g.tokens.to(DEV), g.scores.to(DEV)
            gc = cand.to(DEV)
            ops.beam_prefix(prefix.to(DEV), step, beam, PAD, EOS, gc, V, g)
            OS.beam_prefix(prefix, step, beam, PAD, EOS, cand, V, r)
            assert torch.equal(gc.cpu(), cand) and torch.equal(g.tokens.cpu(), r.tokens) and torch.equal(g.scores.cpu(), r.scores)


def test_diverse_groups_vs_statement():
    from espresso_b200 import ops
    from oracle import search_strategies as OS

    rs = np.random.RandomState(2)
    for V, beam, G, strength in ((5004, 4, 2, 0.5), (5004, 6, 3, 1.3), (5004, 5, 5, 0.3), (13, 4, 1, 0.7), (9, 6, 2, 0.0)):
        bsz = 3
        N = bsz * beam
        lp = torch.from_numpy(np.round(rs.randn(N, V) * 2, 1).astype(np.float32))  # rounded: many exact ties
        lp[0, :] = NEG
        lp[0, 4] = -1.0  # all -inf except one token
        prev = torch.from_numpy(np.round(rs.randn(N), 1).astype(np.float32))
        for step0 in (True, False):
            n_cand = V if step0 else beam // G * V
            Kg = min(2 * (beam // G), n_cand - 1)
            p = None if step0 else prev
            s, t, b = ops.beam_diverse_groups(lp.to(DEV), None if p is None else p.to(DEV), bsz, beam, V, G, Kg, strength)
            sr, tr, br = OS.beam_diverse_groups(lp, p, bsz, beam, V, G, Kg, strength)
            assert torch.equal(s.cpu(), sr) and torch.equal(t.cpu(), tr) and torch.equal(b.cpu(), br), (V, beam, G, step0)
    with pytest.raises(Exception, match="divisible"):
        ops.beam_diverse_groups(lp.to(DEV), None, bsz, 6, 9, 4, 2, 0.5)


def test_sibling_topk_vs_statement():
    from espresso_b200 import ops
    from oracle import search_strategies as OS

    rs = np.random.RandomState(3)
    for V, beam, rate in ((5004, 5, 0.5), (5004, 3, 0.0), (12, 4, 1.1), (6, 2, 0.25)):
        bsz = 4
        N = bsz * beam
        cand = torch.from_numpy(np.round(rs.randn(N, V) * 2, 1).astype(np.float32))
        cand[1, :] = NEG
        cand[1, 3] = 0.5
        k = min(2 * beam, beam * V - 1)
        s, t, b = ops.beam_sibling_topk(cand.to(DEV), bsz, beam, V, k, rate)
        sr, tr, br = OS.beam_sibling_topk(cand, bsz, beam, V, k, rate)
        assert torch.equal(s.cpu(), sr) and torch.equal(t.cpu(), tr) and torch.equal(b.cpu(), br), (V, beam, rate)


class _DevTableModel:
    """tests/test_search_strategies.py's table model with its log-probs on the device."""

    def __init__(self, seed, V):
        from oracle.pin_against_reference import _table_lprobs

        self.fn, self.seed, self.V = _table_lprobs, seed, V

    def max_decoder_positions(self):
        return 40

    def forward_encoder(self, net_input):
        return None

    def init_incremental_state(self, enc, bsz, beam):
        return {}

    def decode_step(self, step, tokens, state, new_order):
        return self.fn(self.seed, self.V, step, tokens.cpu()).to(tokens.device), False


def test_generator_matches_reference_generator_on_gpu(golden_dir):
    from test_search_strategies import _Dict, _fixture, _same
    from oracle.pin_search_strategies import CASES, case_kwargs
    from espresso_b200.sequence_generator import SequenceGenerator

    n = 0
    for c, ref in _fixture(golden_dir):
        m = _DevTableModel(c["seed"], c["V"])
        lm = _DevTableModel(c["seed"] + 1000, c["V"]) if c.get("lm") is not None else None
        gen = SequenceGenerator([m], _Dict(c["V"]), lm_model=lm, lm_weight=c.get("lm") or 1.0, **case_kwargs(c))
        sample = {"net_input": {"src_tokens": torch.zeros(c["bsz"], 7, dtype=torch.long, device=DEV),
                                "src_lengths": torch.full((c["bsz"],), 7, device=DEV)}}
        kw = {"prefix_tokens": torch.tensor(c["prefix"], device=DEV)} if "prefix" in c else {}
        _same(gen.generate([m], sample, **kw), ref, 1e-4)
        n += 1
    assert n == len(CASES)


def _real_model(golden_dir):
    from test_host_orchestration import _build_encdec, _Dict

    g = np.load(os.path.join(golden_dir, "encdec_transformer.npz"))
    m = _build_encdec(g).finalize_(DEV)
    m.eval()

    class D(_Dict):
        def unk(self):
            return 3

    feats, lens = torch.from_numpy(g["feats"]).to(DEV), torch.from_numpy(g["lens"]).to(DEV)
    prefix = torch.from_numpy(g["prev_output_tokens"])[:, 1:3].to(DEV)
    return m, D(50), feats, lens, prefix


OPTIONS = {
    "plain": dict(),
    "ngram": dict(no_repeat_ngram_size=2),
    "groups": dict(diverse_beam_groups=2, diverse_beam_strength=0.5),
    "siblings": dict(diversity_rate=0.5),
    "sampling": dict(sampling=True, sampling_topk=8),
    "prefix": dict(),
}


@pytest.mark.parametrize("name", sorted(OPTIONS))
def test_graph_replay_equals_eager_run(name, golden_dir):
    """Call 1 of a shape runs eagerly, call 2 records one graph per step, later calls replay; every call must agree with a
    generator that never uses graphs, also on new inputs."""
    from espresso_b200.sequence_generator import SequenceGenerator

    m, d, feats, lens, prefix = _real_model(golden_dir)
    kw = dict(beam_size=4, max_len_a=0.5, max_len_b=4, **OPTIONS[name])
    gen = SequenceGenerator([m], d, **kw)
    eager = SequenceGenerator([m], d, use_cuda_graphs=False, **kw)
    pkw = {"prefix_tokens": prefix} if name == "prefix" else {}
    torch.manual_seed(11)
    feats2 = feats.roll(1, dims=0) + 0.3 * torch.randn_like(feats)
    for inp in (feats, feats, feats2, feats):
        smp = {"net_input": {"src_tokens": inp, "src_lengths": lens}}
        hg, he = gen.generate([m], smp, **pkw), eager.generate([m], smp, **pkw)
        for a, b in zip(hg, he):
            assert len(a) == len(b) >= 1
            for x, y in zip(a, b):
                assert x["tokens"].tolist() == y["tokens"].tolist()
                assert abs(float(x["score"]) - float(y["score"])) < 1e-5
    assert len(next(iter(gen._graph_cache.values()))["graphs"]) > 0


def test_launches_per_step(golden_dir):
    """Search launches per step, counted between the end of one decoder step and the start of the next: plain beam search
    keeps the parent's 3 (esp_beam_merge, esp_beam_topk, esp_beam_bookkeep); n-gram blocking and a forced prefix add one
    each where they apply; diverse groups and sampling keep 3; diverse siblings take 6 after step 0 (merge, row top-k,
    penalty, pool top-k, remap, bookkeeping)."""
    from espresso_b200 import lib
    from espresso_b200.sequence_generator import SequenceGenerator

    m, d, feats, lens, prefix = _real_model(golden_dir)
    marks = []
    orig = m.decode_step

    def counted(step, tokens, state, new_order):
        marks.append(lib.launch_count())
        out = orig(step, tokens, state, new_order)
        marks.append(lib.launch_count())
        return out

    def per_step(pkw=None, **kw):
        marks.clear()
        m.decode_step = counted
        try:
            gen = SequenceGenerator([m], d, beam_size=4, max_len_a=0.5, max_len_b=4, use_cuda_graphs=False, **kw)
            gen.generate([m], {"net_input": {"src_tokens": feats, "src_lengths": lens}}, **(pkw or {}))
        finally:
            m.decode_step = orig
        assert len(marks) >= 6
        return [marks[2 * t + 2] - marks[2 * t + 1] for t in range(len(marks) // 2 - 1)]

    plain = per_step()
    assert plain == [3] * len(plain)
    ngram = per_step(no_repeat_ngram_size=2)
    assert ngram == [3] + [4] * (len(ngram) - 1)  # nothing to block at step 0
    assert per_step(diverse_beam_groups=2) == [3] * len(per_step(diverse_beam_groups=2))
    sib = per_step(diversity_rate=0.5)
    assert sib == [3] + [6] * (len(sib) - 1)  # step 0 is plain beam search
    smp = per_step(sampling=True, sampling_topk=5)
    assert smp == [3] * len(smp)
    pre = per_step(pkw={"prefix_tokens": prefix})  # forced at steps 0 and 1
    assert pre[:2] == [4, 4] and pre[2:] == [3] * (len(pre) - 2)


def test_sample_vs_statement():
    from espresso_b200 import ops
    from oracle import search_strategies as OS

    rs = np.random.RandomState(4)
    for V, beam, bsz in ((5004, 5, 3), (37, 4, 3), (9, 2, 4)):
        N = bsz * beam
        lp = torch.log_softmax(torch.from_numpy(np.round(rs.randn(N, V) * 2, 1).astype(np.float32)), -1)  # ties
        lp[0, :] = NEG
        lp[0, 6] = -0.3  # one finite token
        lp[1, :] = NEG   # no mass at all
        prev = torch.from_numpy(rs.randn(N).astype(np.float32))
        for topk, topp in ((-1, -1.0), (1, -1.0), (7, -1.0), (-1, 0.3), (-1, 0.9), (-1, 1.0), (V + 3, -1.0)):
            for step, p in ((0, None), (5, prev)):
                seed = torch.tensor([12345 + step], dtype=torch.int64)
                s, t, b = ops.beam_sample(lp.to(DEV), None if p is None else p.to(DEV), bsz, beam, V, topk, topp, seed.to(DEV), step)
                sr, tr, br = OS.beam_sample(lp, p, bsz, beam, V, topk, topp, seed, step)
                assert torch.equal(t.cpu(), tr) and torch.equal(b.cpu(), br), (V, topk, topp, step)
                fin = torch.isfinite(sr)
                assert torch.equal(torch.isfinite(s.cpu()), fin)
                assert (s.cpu()[fin] - sr[fin]).abs().max().item() < 1e-5, (V, topk, topp, step)


@pytest.mark.parametrize("topk,topp", [(-1, -1.0), (12, -1.0), (-1, 0.7)])
def test_sample_chi_square(topk, topp):
    """2^20 draws from one row against the truncated, renormalised distribution."""
    from scipy import stats

    from espresso_b200 import ops

    V, bsz, beam = 40, 1024, 4  # 4096 draws per launch, 256 launches
    lp = torch.log_softmax(torch.from_numpy(np.random.RandomState(5).randn(V).astype(np.float32)) * 1.5, -1)
    rows = lp[None].repeat(bsz * beam, 1).contiguous().to(DEV)
    prev = torch.zeros(bsz * beam, device=DEV)
    counts = torch.zeros(V, dtype=torch.int64, device=DEV)
    seed = torch.tensor([77], dtype=torch.int64, device=DEV)
    for step in range(1, 257):
        _, t, _ = ops.beam_sample(rows, prev, bsz, beam, V, topk, topp, seed, step)
        counts += torch.bincount(t.reshape(-1).long(), minlength=V)
    counts = counts.cpu().double()
    assert int(counts.sum()) == 2 ** 20
    # the kept set and its masses, from the statement's rule
    p = torch.exp(lp).numpy()
    W = np.array([int(np.float32(x) * np.float32(2.0 ** 40)) for x in p], dtype=np.float64)
    order = sorted(range(V), key=lambda v: (-float(p[v]), v))
    keep = np.ones(V, bool)
    if topp > 0 or topk > 0:
        limit = int(np.float32(topp) * np.float32(2.0 ** 40)) if topp > 0 else topk
        before = 0
        for v in order:
            keep[v] = before < limit
            before += int(W[v]) if topp > 0 else 1
    assert counts[torch.from_numpy(~keep)].sum() == 0
    exp = W[keep] / W[keep].sum() * 2 ** 20
    chi2 = float(((counts.numpy()[keep] - exp) ** 2 / exp).sum())
    assert chi2 < stats.chi2.ppf(1 - 1e-6, int(keep.sum()) - 1), chi2


def test_sampling_seed_advances_and_replays(golden_dir):
    """The seed lives in device memory: graph replays draw fresh samples on every call, equal to an eager generator's
    with the same seed; the same seed gives the same hypotheses."""
    from espresso_b200.sequence_generator import SequenceGenerator

    m, d, feats, lens, _ = _real_model(golden_dir)
    kw = dict(beam_size=4, max_len_a=0.5, max_len_b=4, sampling=True, sampling_topp=0.95, sampling_seed=3)
    gen, eager = SequenceGenerator([m], d, **kw), SequenceGenerator([m], d, use_cuda_graphs=False, **kw)
    smp = {"net_input": {"src_tokens": feats, "src_lengths": lens}}
    calls = []
    for _ in range(4):
        hg, he = gen.generate([m], smp), eager.generate([m], smp)
        tg = [[x["tokens"].tolist() for x in a] for a in hg]
        assert tg == [[x["tokens"].tolist() for x in a] for a in he]
        calls.append(tg)
    assert len(next(iter(gen._graph_cache.values()))["graphs"]) > 0
    assert any(c != calls[0] for c in calls[1:])  # fresh draws per call
