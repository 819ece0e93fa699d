"""CPU: fairseq's search options in the native SequenceGenerator -- diverse beam search, diverse siblings, sampling,
n-gram blocking and forced prefixes.

  * the oracle (oracle/search_strategies.py) against the real reference's hypotheses recorded by
    oracle/pin_search_strategies.py (tests/golden/search_strategies.npz) and against the reference's own known answers
    (TestDiverseBeamSearch, TestDiverseSiblingsSearch, TestTopPSamplingSearch, TestRepeatNgramBlocking in
    tests/test_sequence_generator.py);
  * the product generator's host orchestration, with the per-op statements monkeypatched in for the kernels, against the
    fixture, the known answers and the oracle on random table models;
  * the option plumbing of the task's build_generator and of recognize(), including the reference's refusals.
The kernels themselves are checked against the same per-op statements in test_gpu_search_strategies.py."""
import math
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

from oracle import ops_ref
from oracle import search_strategies as OS
from oracle.pin_against_reference import _table_lprobs
from oracle.pin_search_strategies import CASES, case_kwargs, lprobs_fn

PAD, EOS, UNK, W1, W2 = 1, 2, 3, 4, 5
NEG_INF = float("-inf")


class _Dict:
    def __init__(self, V):
        self.V = V

    def __len__(self):
        return self.V

    def pad(self):
        return PAD

    def eos(self):
        return EOS

    def unk(self):
        return UNK


@pytest.fixture()
def cpu_ops(monkeypatch):
    from espresso_b200 import ops

    for mod in (ops_ref, OS):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                monkeypatch.setattr(ops, name, getattr(mod, name))
    return ops


class _TableModel:
    """The pin's prefix-dependent table model (optionally with the LM table added) behind the generator's model protocol."""

    def __init__(self, seed, V, lm=None):
        self.seed, self.V, self.lm = seed, V, lm

    def max_decoder_positions(self):
        return 40

    def forward_encoder(self, net_input):
        return None

    def init_incremental_state(self, enc, bsz, beam):
        return {}

    def decode_step(self, step, tokens, state, new_order):
        return _table_lprobs(self.seed, self.V, step, tokens), False


def _fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "search_strategies.npz"))
    assert int(g["n_cases"]) == len(CASES)
    for ci, c in enumerate(CASES):
        ref = [[(g["c%d_b%d_k%d_tokens" % (ci, b, k)].tolist(), float(g["c%d_b%d_k%d_score" % (ci, b, k)]))
                for k in range(int(g["c%d_b%d_n" % (ci, b)]))] for b in range(c["bsz"])]
        yield c, ref


def _product(c, **extra):
    from espresso_b200.sequence_generator import SequenceGenerator

    m = _TableModel(c["seed"], c["V"])
    lm = _TableModel(c["seed"] + 1000, c["V"]) if c.get("lm") is not None else None
    gen = SequenceGenerator([m], _Dict(c["V"]), lm_model=lm, lm_weight=c.get("lm") or 1.0, **case_kwargs(c), **extra)
    sample = {"net_input": {"src_tokens": torch.zeros(c["bsz"], 7, dtype=torch.long), "src_lengths": torch.full((c["bsz"],), 7)}}
    kw = {"prefix_tokens": torch.tensor(c["prefix"])} if "prefix" in c else {}
    return gen.generate([m], sample, **kw)


def _same(got, ref, tol):
    assert len(got) == len(ref)
    for hs, rs in zip(got, ref):
        assert len(hs) == len(rs)
        for h, (toks, score) in zip(hs, rs):
            assert h["tokens"].tolist() == toks, (h["tokens"].tolist(), toks)
            assert abs(float(h["score"]) - score) < tol


def test_oracle_matches_reference_generator(golden_dir):
    for c, ref in _fixture(golden_dir):
        prefix = torch.tensor(c["prefix"]) if "prefix" in c else None
        got = OS.generate(lprobs_fn(c), c["bsz"], 7, c["V"], PAD, UNK, EOS, model_max_len=40, prefix_tokens=prefix, **case_kwargs(c))
        _same(got, ref, 1e-5)


def test_product_matches_reference_generator(golden_dir, cpu_ops):
    for c, ref in _fixture(golden_dir):
        _same(_product(c), ref, 1e-4)


def test_fixture_cases_differ_from_plain_beam_search(golden_dir):
    """Every option in the fixture changes the hypotheses (otherwise it would pin nothing)."""
    from oracle import beam as OB

    for c, ref in _fixture(golden_dir):
        kw = {k: v for k, v in case_kwargs(c).items() if k in ("beam_size", "max_len_a", "max_len_b", "min_len", "len_penalty",
                                                                 "unk_penalty", "eos_factor")}
        plain = OB.generate(lprobs_fn(c), c["bsz"], 7, c["V"], PAD, UNK, EOS, model_max_len=40, **kw)
        assert [[h["tokens"].tolist() for h in hs] for hs in plain] != [[t for t, _ in rs] for rs in ref], c


# ---------------------------------------------------------------------------------------------------------------------
# the reference's known answers (tests/test_sequence_generator.py:330-564, tables as in TestDiverseBeamSearch.setUp)
# ---------------------------------------------------------------------------------------------------------------------
DIVERSE_PROBS = [
    torch.tensor([[0.0, 0.0, 0.9, 0.1], [0.0, 0.0, 0.9, 0.1], [0.0, 0.0, 0.7, 0.3], [0.0, 0.0, 0.7, 0.3]]),
    torch.tensor([[0.0, 0.0, 0.6, 0.4], [0.0, 0.0, 0.6, 0.4], [0.25, 0.0, 0.35, 0.4], [0.25, 0.0, 0.35, 0.4]]),
    torch.tensor([[1.0, 0.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.0], [0.9, 0.0, 0.1, 0.0], [0.9, 0.0, 0.1, 0.0]]),
]


def _known(kind, product):
    kw = dict(diverse_beam_groups=2, diverse_beam_strength=0.0) if kind == "groups" else dict(diversity_rate=0.5)
    if product:
        from espresso_b200.sequence_generator import SequenceGenerator, TableDecoderModel

        m = TableDecoderModel(DIVERSE_PROBS, 6, EOS)
        g = SequenceGenerator([m], _Dict(6), beam_size=2, **kw)
        sample = {"net_input": {"src_tokens": torch.tensor([[W1, W2, EOS]] * 2), "src_lengths": torch.tensor([2, 2])}}
        return g.generate([m], sample)

    def fn(step, tokens, ro):
        probs = torch.zeros(tokens.shape[0], 6)
        if step < len(DIVERSE_PROBS):
            probs[:, EOS:] = DIVERSE_PROBS[step][: tokens.shape[0]]
        else:
            probs[:, EOS] = 1.0
        return probs.log()

    return OS.generate(fn, 2, 3, 6, PAD, UNK, EOS, beam_size=2, **kw)


def _check(h, toks, probs, ranks=None, rate=0.0):
    assert h["tokens"].tolist() == toks
    ps = torch.tensor(probs).log()
    if ranks is not None:
        ps = ps - torch.tensor(ranks, dtype=torch.float32) * rate
    assert (h["positional_scores"] - ps).abs().max() < 1e-4
    assert abs(float(ps.sum() / len(probs)) - float(h["score"])) < 1e-4


@pytest.mark.parametrize("product", [False, True])
def test_known_answers_diverse_beam_search(product, request):
    if product:
        request.getfixturevalue("cpu_ops")
    h = _known("groups", product)
    _check(h[0][0], [W1, W1, EOS], [0.9, 0.6, 1.0])
    _check(h[0][1], [W1, W1, EOS], [0.9, 0.6, 1.0])
    _check(h[1][0], [W1, W2, EOS], [0.7, 0.4, 0.9])
    _check(h[1][1], [W1, W2, EOS], [0.7, 0.4, 0.9])


@pytest.mark.parametrize("product", [False, True])
def test_known_answers_diverse_siblings_search(product, request):
    if product:
        request.getfixturevalue("cpu_ops")
    h = _known("siblings", product)
    _check(h[0][0], [W1, W1, EOS], [0.9, 0.6, 1.0], [0, 1, 1], 0.5)
    _check(h[0][1], [W1, W2, EOS], [0.9, 0.4, 1.0], [0, 2, 1], 0.5)
    _check(h[1][0], [W1, W2, EOS], [0.7, 0.4, 0.9], [0, 1, 1], 0.5)
    _check(h[1][1], [W1, W1, EOS], [0.7, 0.35, 0.9], [0, 2, 1], 0.5)


TOPP_PROBS = [  # TestTopPSamplingSearch.setUp: min top-1 probability 0.4, min top-2 probability 0.75
    torch.tensor([[0.0, 0.0, 1.0, 0.0]] * 4),
    torch.tensor([[0.25, 0.0, 0.4, 0.35]] * 4),
    torch.tensor([[1.0, 0.0, 0.0, 0.0]] * 4),
]


@pytest.mark.parametrize("product", [False, True])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_known_answers_top_p_sampling(product, seed, request):
    """TestTopPSamplingSearch: p = 0.2 keeps only the top token; p = 0.575 keeps the top two."""
    from espresso_b200.sequence_generator import SequenceGenerator, TableDecoderModel

    if product:
        request.getfixturevalue("cpu_ops")
    seen = set()
    for topp in (0.2, 0.575):
        kw = dict(sampling=True, sampling_topp=topp, sampling_seed=seed)
        if product:
            m = TableDecoderModel(TOPP_PROBS, 6, EOS)
            g = SequenceGenerator([m], _Dict(6), beam_size=2, **kw)
            sample = {"net_input": {"src_tokens": torch.tensor([[W1, W2, EOS]] * 2), "src_lengths": torch.tensor([2, 2])}}
            h = g.generate([m], sample)
        else:
            def fn(step, tokens, ro):
                probs = torch.zeros(tokens.shape[0], 6)
                probs[:, EOS:] = TOPP_PROBS[step][: tokens.shape[0]] if step < 3 else torch.tensor([1.0, 0, 0, 0])
                return probs.log()

            h = OS.generate(fn, 2, 3, 6, PAD, UNK, EOS, beam_size=2, **kw)
        for hs in h:
            for x in hs:
                if topp == 0.2:
                    _check(x, [W1, W1, EOS], [1.0, 0.4, 1.0])
                else:
                    assert x["tokens"].tolist() in ([W1, W1, EOS], [W1, W2, EOS])
                    _check(x, x["tokens"].tolist(), [1.0, 0.4 if x["tokens"][1] == W1 else 0.35, 1.0])
                    seen.add(int(x["tokens"][1]))
    assert seen  # the high-p draws land on the two kept tokens only


def test_sampling_statement_edges():
    """esp_beam_sample's statement: top-k = 1 is the arg-max (lowest token on ties), tiny top-p keeps the top token, a row
    with one finite token always draws it, and a row without mass gives token 0 at -inf."""
    lp = torch.log_softmax(torch.tensor([[0.0, 2.0, 2.0, -1.0, 1.0]] * 4), -1)
    s, t, b = OS.beam_sample(lp, None, 2, 2, 5, 1, -1.0, 9, 0)
    assert t.tolist() == [[1, 1], [1, 1]] and b.tolist() == [[0, 0], [0, 0]]
    s, t, b = OS.beam_sample(lp, torch.arange(4.0), 2, 2, 5, -1, 1e-3, 9, 3)
    assert t.tolist() == [[1, 1], [1, 1]] and b.tolist() == [[0, 1], [0, 1]]
    assert torch.allclose(s, torch.log(torch.exp(lp[:, 1])).view(2, 2) + torch.arange(4.0).view(2, 2))
    one = torch.full((2, 5), NEG_INF)
    one[0, 3] = -0.2
    s, t, _ = OS.beam_sample(one, torch.zeros(2), 1, 2, 5, -1, -1.0, 9, 1)
    assert t.tolist() == [[3, 0]] and float(s[0, 1]) == NEG_INF


def test_known_answer_repeat_ngram_blocking():
    """TestRepeatNgramBlocking.test_finds_repetitive_tokens: n = 2, step 3."""
    lp = torch.zeros(2, 4)
    OS.beam_block_ngrams(torch.tensor([[2, 2, 2, 2], [3, 3, 3, 3]], dtype=torch.int32), 3, 2, lp, 4)
    assert lp.tolist() == [[0.0, 0.0, -math.inf, 0.0], [0.0, 0.0, 0.0, -math.inf]]


def test_ngram_statement_matches_reference_fallback_rule():
    """The reference's Python rule (_no_repeat_ngram over a step + 1 column history), restated literally, on random
    histories (TestRepeatNgramBlocking.test_ngram_blocking_same_as_default_implem, n = 2..4)."""
    rs = np.random.RandomState(5)
    for _ in range(40):
        n, step, rows, V = int(rs.randint(2, 5)), int(rs.randint(0, 9)), 3, 5
        toks = rs.randint(0, V, size=(rows, step + 1))
        got = OS.beam_block_ngrams(torch.from_numpy(toks).int(), step, n, torch.zeros(rows, V), V)
        want = torch.zeros(rows, V)
        if step + 2 - n >= 0:
            for r in range(rows):
                row = toks[r].tolist()
                for i in range(step + 2 - n):
                    if row[-(n - 1):] == row[i: i + n - 1]:
                        want[r, row[i + n - 1]] = -math.inf
        assert torch.equal(got, want)


# ---------------------------------------------------------------------------------------------------------------------
# product vs oracle on random table models (beyond the fixture's shapes)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opts", [
    dict(seed=51, beam=4, bsz=3, V=15, groups=4, strength=0.8),
    dict(seed=52, beam=6, bsz=2, V=9, groups=2, strength=2.0, eos_factor=1.5, ngram=3),
    dict(seed=53, beam=5, bsz=3, V=14, rate=0.9, ngram=2),
    dict(seed=54, beam=2, bsz=4, V=8, ngram=2, groups=2, strength=0.5),
    dict(seed=55, beam=4, bsz=3, V=12, ngram=4, prefix=[[4, 4, 4, 5, 6], [6, EOS, PAD, PAD, PAD], [PAD, 7, PAD, 9, PAD]]),
    dict(seed=56, beam=4, bsz=3, V=11, topp=0.8),
    dict(seed=57, beam=3, bsz=4, V=14, topk=4, ngram=2),
    dict(seed=58, beam=2, bsz=3, V=9, topk=-1, topp=-1.0, prefix=[[5, EOS], [PAD, 6], [7, PAD]]),
])
def test_product_matches_oracle_on_random_models(opts, cpu_ops):
    """Sampled tokens too: the product draws with the same seed sequence as the oracle (sampling_seed = 1, +1 per call)."""
    c = dict(opts)
    got = _product(c)
    prefix = torch.tensor(c["prefix"]) if "prefix" in c else None
    ref = OS.generate(lprobs_fn(c), c["bsz"], 7, c["V"], PAD, UNK, EOS, model_max_len=40, prefix_tokens=prefix, **case_kwargs(c))
    for hs, rs in zip(got, ref):
        assert len(hs) == len(rs)
        for h, r in zip(hs, rs):
            assert h["tokens"].tolist() == r["tokens"].tolist()
            assert abs(float(h["score"]) - float(r["score"])) < 1e-5
            assert (h["positional_scores"] - r["positional_scores"]).abs().max() < 1e-5


def test_fairseq_search_objects_map_to_the_keywords(cpu_ops):
    """A fairseq search object passed as search_strategy selects the same search as the keywords."""
    from espresso_b200.sequence_generator import SequenceGenerator

    class DiverseBeamSearch:
        num_groups, diversity_strength = 2, -0.7  # fairseq stores the negated strength

    class DiverseSiblingsSearch:
        diversity_rate = 0.4

    class Sampling:
        sampling_topk, sampling_topp = 5, -1.0

    class LexicallyConstrainedBeamSearch:
        pass

    m = _TableModel(1, 9)
    g = SequenceGenerator([m], _Dict(9), beam_size=4, search_strategy=DiverseBeamSearch())
    assert (g.diverse_beam_groups, g.diverse_beam_strength, g.diversity_rate) == (2, 0.7, -1.0)
    g = SequenceGenerator([m], _Dict(9), beam_size=4, search_strategy=DiverseSiblingsSearch())
    assert (g.diverse_beam_groups, g.diversity_rate) == (-1, 0.4)
    g = SequenceGenerator([m], _Dict(9), beam_size=4, search_strategy=Sampling())
    assert (g.sampling, g.sampling_topk, g.sampling_topp) == (True, 5, -1.0)
    with pytest.raises(NotImplementedError, match="LexicallyConstrainedBeamSearch"):
        SequenceGenerator([m], _Dict(9), beam_size=4, search_strategy=LexicallyConstrainedBeamSearch())


# ---------------------------------------------------------------------------------------------------------------------
# option plumbing and refusals
# ---------------------------------------------------------------------------------------------------------------------
def _task():
    from espresso_b200.data.asr_dictionary import AsrDictionary
    from espresso_b200.tasks.speech_recognition import SpeechRecognitionEspressoConfig, SpeechRecognitionEspressoTask

    d = AsrDictionary()
    for ch in "abcdefgh":
        d.add_symbol(ch)
    return SpeechRecognitionEspressoTask(SpeechRecognitionEspressoConfig(criterion_name="label_smoothed_cross_entropy_v2"), d,
                                         feat_dim=80)


def test_build_generator_reads_the_search_options():
    task, m = _task(), _TableModel(1, 9)
    g = task.build_generator([m], Namespace(beam=4, no_repeat_ngram_size=3, diverse_beam_groups=2, diverse_beam_strength=0.2))
    assert (g.no_repeat_ngram_size, g.diverse_beam_groups, g.diverse_beam_strength, g.diversity_rate) == (3, 2, 0.2, -1.0)
    g = task.build_generator([m], Namespace(beam=4, diversity_rate=0.0))
    assert (g.diverse_beam_groups, g.diversity_rate) == (-1, 0.0)
    g = task.build_generator([m], Namespace(beam=4, sampling=True, sampling_topp=0.9, seed=7))
    assert (g.sampling, g.sampling_topk, g.sampling_topp, g._next_seed, g.diversity_rate) == (True, -1, 0.9, 7, -1.0)
    g = task.build_generator([m], Namespace(beam=4, match_source_len=True, diversity_rate=0.0))  # checked before siblings
    assert g.diversity_rate == -1.0
    g = task.build_generator([m], Namespace(beam=4))  # no option: plain beam search, as before
    assert (g.no_repeat_ngram_size, g.diverse_beam_groups, g.diversity_rate) == (0, -1, -1.0)


@pytest.mark.parametrize("args,exc,msg", [
    (dict(diverse_beam_groups=2, diversity_rate=0.5), ValueError, "mutually exclusive"),
    (dict(sampling=True, diverse_beam_groups=2), ValueError, "mutually exclusive"),
    (dict(sampling=True, diversity_rate=0.3), ValueError, "mutually exclusive"),
    (dict(sampling_topk=5), AssertionError, "--sampling-topk requires --sampling"),
    (dict(sampling_topp=0.9), AssertionError, "--sampling-topp requires --sampling"),
    (dict(diverse_beam_groups=3), ValueError, "divisible by the number of groups"),
])
def test_build_generator_refusals(args, exc, msg):
    with pytest.raises(exc, match=msg):
        _task().build_generator([_TableModel(1, 9)], Namespace(beam=4, **args))


def test_recognize_requires_nbest_equal_to_beam_under_sampling():
    from espresso_b200.speech_recognize import recognize

    with pytest.raises(AssertionError, match="--sampling requires --nbest to be equal to --beam"):
        recognize(None, [], gen_args=Namespace(sampling=True, beam=5), nbest=1)


def test_recognize_forces_the_target_prefix(monkeypatch):
    """recognize() hands the first prefix_size target tokens of each batch to the generator (speech_recognize.py:246-248)."""
    from espresso_b200 import speech_recognize as SR

    seen = []

    class Gen:
        def generate(self, models, sample, **kw):
            seen.append(kw)
            return [[{"tokens": torch.tensor([4, EOS]), "score": torch.tensor(0.0), "attention": None}]] * len(sample["id"])

    class Model(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(1))

    task = _task()
    batch = {"id": torch.tensor([0, 1]), "utt_id": ["u0", "u1"], "net_input": {"src_tokens": torch.zeros(2, 5, 80)},
             "target": torch.tensor([[5, 6, 7, EOS], [8, EOS, PAD, PAD]])}
    monkeypatch.setattr(task, "build_generator", lambda models, args, extra_gen_cls_kwargs=None: Gen())
    monkeypatch.setattr(task, "load_dataset", lambda subset: None)
    monkeypatch.setattr(task, "dataset", lambda subset: None)
    task.datasets["test"] = None

    class Itr:
        def next_epoch_itr(self, shuffle=False):
            return iter([batch])

    monkeypatch.setattr(task, "get_batch_iterator", lambda *a, **k: Itr())
    SR.recognize(task, [Model()], subset="test", gen_args=Namespace(prefix_size=2), device="cpu")
    assert seen[-1]["prefix_tokens"].tolist() == [[5, 6], [8, EOS]]
    SR.recognize(task, [Model()], subset="test", gen_args=Namespace(), device="cpu")
    assert seen[-1] == {}
