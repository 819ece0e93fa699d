"""CPU: ARPA n-gram LMs and the CTC search fused with them.  oracle/ngram.py (float64 backoff recursion over full
histories, a seeded normalised ARPA writer, the lexicon search statement) is pinned by hand-worked values, by
normalisation and by exhaustive enumeration; the host builder behind esp_ngram_build is pinned against it through the
fp32 restatement of the kernels' walk (oracle/ctc_ngram_ops.probe); the host orchestration of CTCDecoder runs over
oracle/ops_ref + ctc_beam_ops + ctc_ngram_ops and must reproduce the oracle, lexicon-free and through a lexicon."""
import gzip
import itertools
import math
from argparse import Namespace

import numpy as np
import pytest
import torch

from oracle import ctc_beam as O
from oracle import ngram as N
from oracle.ctc_ngram_ops import probe, state_of
from test_ctc_beam_search import _FakeCTC, _ctc_logp, _dict, _enumerate, _logits, _task

TOY = """\\data\\
ngram 1=6
ngram 2=4
ngram 3=2

\\1-grams:
-1.0\t<unk>\t0.0
-99\t<s>\t-0.5
-0.7\t</s>
-0.9\ta\t-0.3
-1.1\tb\t-0.2
-1.3\tc\t-0.25

\\2-grams:
-0.4\t<s> a\t-0.15
-0.6\ta b\t-0.1
-0.5\tb c
-0.8\ta </s>

\\3-grams:
-0.2\t<s> a b
-0.3\ta b c

\\end\\
"""


def _load(tmp_path, text, name="lm.arpa"):
    from espresso_b200.models import NgramLanguageModel

    p = tmp_path / name
    if name.endswith(".gz"):
        with gzip.open(p, "wt") as f:
            f.write(text)
    else:
        p.write_text(text)
    return NgramLanguageModel.from_arpa(str(p))


def test_oracle_scorer_known_answers(tmp_path):
    (tmp_path / "toy.arpa").write_text(TOY)
    a = N.Arpa.read(tmp_path / "toy.arpa")
    # listed trigram; a backoff chain of depth N - 1 = 2: bo(a b) + bo(b) + p(a)
    assert a.logp(["<s>", "a"], "b") == pytest.approx(-0.2)
    assert a.logp(["a", "b"], "a") == pytest.approx(-0.1 - 0.2 - 0.9)
    # unlisted context (c a): backoff 0, then bo(a) + p(c)
    assert a.logp(["c", "a"], "c") == pytest.approx(-0.3 - 1.3)
    # <unk>: unknown words score as <unk>, also in the history
    assert a.logp(["<s>"], "zzz") == pytest.approx(-0.5 - 1.0)
    assert a.logp(["zzz"], "a") == pytest.approx(-0.9)
    # </s>, and a sentence
    assert a.logp(["<s>", "a"], "</s>") == pytest.approx(-0.15 - 0.8)
    # (b c) listed without a backoff: 0, then bo(c) + p(</s>)
    assert a.sentence_logp(["a", "b", "c"]) == pytest.approx(-0.4 - 0.2 - 0.3 + (0.0 - 0.25 - 0.7))
    # without <unk>: -100, as KenLM
    (tmp_path / "nounk.arpa").write_text(TOY.replace("ngram 1=6", "ngram 1=5").replace("-1.0\t<unk>\t0.0\n", ""))
    b = N.Arpa.read(tmp_path / "nounk.arpa")
    assert b.logp(["b"], "zzz") == pytest.approx(-0.2 - 100.0)


@pytest.mark.parametrize("order", [2, 3, 4, 5])
def test_oracle_writer_is_normalised(tmp_path, order):
    a = N.write_arpa(tmp_path / "w.arpa", order, n_words=14, n_sent=120, seed=order)
    vocab = [w for w in a.vocab if w != "<s>"]
    rs = np.random.RandomState(order)
    hists = [["<s>"]] + [["<s>"] + [vocab[i] for i in rs.randint(0, len(vocab), size=rs.randint(1, order + 1))]
                          for _ in range(30)]
    hists += [["<s>", "w0", "w1", "w0"][:order], ["w5", "w5", "w5", "w5"]]  # seen and unseen
    for h in hists:
        assert abs(sum(10.0 ** a.logp(h, w) for w in vocab) - 1.0) < 1e-9, h


def _random_pairs(a, n, seed, order):
    rs = np.random.RandomState(seed)
    words = a.vocab + ["oov"]
    out = []
    for _ in range(n):
        h = ["<s>"] + [words[i] for i in rs.randint(0, len(words), size=rs.randint(0, order + 1))]
        out.append((h, words[rs.randint(0, len(words))]))
    return out


@pytest.mark.parametrize("order", [1, 2, 3, 4, 5, 6])
def test_host_builder_matches_the_oracle(tmp_path, order):
    a = N.write_arpa(tmp_path / "w.arpa", order, n_words=25, n_sent=250, seed=10 + order)
    lm = _load(tmp_path, (tmp_path / "w.arpa").read_text())
    assert lm.order == order and lm.vocab == a.vocab
    assert lm.counts == [len(g) for g in a.grams]
    n = 100000 // 6
    err = 0.0
    for h, w in _random_pairs(a, n, order, order):
        s = state_of(lm, [lm.index(x) for x in h[1:]])
        lp, nxt = probe(lm, s, lm.index(w))
        ref = a.logp(h, w)
        err = max(err, abs(float(lp) - ref) / max(1.0, abs(ref)))
        # the next state is the longest listed suffix of (history + w), of order < N
        hw = tuple(a._known(x) for x in h + [w])
        want = -1
        for k in range(min(order - 1, len(hw)), 0, -1):
            if hw[len(hw) - k:] in a.grams[k - 1]:
                want = k
                break
        got = () if nxt < 0 else _entry_words(lm, nxt)
        assert got == (hw[len(hw) - want:] if want > 0 else ()), (h, w, got)
    assert err < 1e-6


def _entry_words(lm, e):
    """The words of table entry e, read back through the tables (its context chain)."""
    ws = [lm.vocab[lm.word[e]]]
    order = int(np.searchsorted(lm.order_off, e, side="right"))
    while order > 1:
        lo = lm.order_off[order - 2]
        # the parent is the entry of order - 1 whose child range holds e
        cand = np.flatnonzero((lm.child_lo[lo:lm.order_off[order - 1]] <= e) & (lm.child_hi[lo:lm.order_off[order - 1]] > e))
        e = int(lo + cand[0])
        ws.insert(0, lm.vocab[lm.word[e]])
        order -= 1
    return tuple(ws)


def test_host_builder_refusals_gz_and_stable_ids(tmp_path):
    from espresso_b200.lib import EspressoB200Error

    lm = _load(tmp_path, TOY)
    lz = _load(tmp_path, TOY, "lm.arpa.gz")
    assert lm.vocab == lz.vocab == ["<unk>", "<s>", "</s>", "a", "b", "c"]
    for k in ("word", "prob", "backoff", "child_lo", "child_hi", "suffix"):
        assert np.array_equal(getattr(lm, k), getattr(lz, k))
    assert lm.index("b") == 4 and lm.index("nope") == lm.unk == 0 and lm.eos == 2 and lm.start == 1
    nounk = _load(tmp_path, TOY.replace("ngram 1=6", "ngram 1=5").replace("-1.0\t<unk>\t0.0\n", ""), "n.arpa")
    assert nounk.unk_added and nounk.vocab[-1] == "<unk>" and nounk.prob[nounk.unk] == -100.0
    assert nounk.vocab[:-1] == ["<s>", "</s>", "a", "b", "c"]
    bad = {
        "KenLM binary": "mmap lm http://kheafield.com/code format version 5\0\0\0",
        "context of this 3-gram is not listed": TOY.replace("-0.3\ta b c", "-0.3\tb a c"),
        "positive log-probability 0.5 at line 16": TOY.replace("-0.6\ta b\t-0.1", "0.5\ta b\t-0.1"),
        "malformed 2-gram at line 17": TOY.replace("-0.5\tb c", "-0.5\tb c d e"),
        "malformed log-probability at line 10": TOY.replace("-0.9\ta", "x\ta"),
        "header says": TOY.replace("ngram 2=4", "ngram 2=5"),
        "not among the 1-grams": TOY.replace("-0.5\tb c", "-0.5\tb q"),
        "order 7": TOY.replace("ngram 3=2", "ngram 3=2\nngram 4=0\nngram 5=0\nngram 6=0\nngram 7=0"),
    }
    for msg, text in bad.items():
        with pytest.raises(EspressoB200Error, match=msg):
            _load(tmp_path, text, "bad.arpa")


def test_host_builder_reads_compact_headers(tmp_path):
    """Hand-edited layouts: the 1-grams right after the counts, trailing whitespace on section lines."""
    lm = _load(tmp_path, TOY)
    compact = TOY.replace("ngram 3=2\n\n\\1-grams:", "ngram 3=2\n\\1-grams:").replace("\\data\\\n", "\\data\\ \t\n")
    compact = compact.replace("\\2-grams:\n", "\\2-grams:  \n")
    assert compact != TOY
    lc = _load(tmp_path, compact, "compact.arpa")
    assert lc.vocab == lm.vocab and lc.counts == lm.counts
    for k in ("word", "prob", "backoff", "child_lo", "child_hi", "suffix"):
        assert np.array_equal(getattr(lm, k), getattr(lc, k))


# ---- searches -------------------------------------------------------------------------------------------------------
def _sym_arpa(tmp_path, d, order, seed):
    """An ARPA over the dictionary's piece symbols (lexicon-free mode)."""
    pieces = [d[i] for i in range(d.nspecial, len(d))]
    return N.write_arpa(tmp_path / "sym.arpa", order, n_words=len(pieces), n_sent=200, seed=seed, words=pieces)


@pytest.mark.parametrize("lm_weight,word_score,order", [(0.47, 0.0, 2), (0.8, -0.3, 3), (1.3, 0.7, 4)])
def test_lexicon_free_oracle_is_the_closed_form(tmp_path, lm_weight, word_score, order):
    d = _dict(n_sym=3)
    V, blank, eos = len(d), 0, d.eos()
    a = _sym_arpa(tmp_path, d, order, seed=order)
    sym = lambda y: [d[v] for v in y]  # noqa: E731

    def lm_fn(y):
        return np.array([a.logp(["<s>"] + sym(y), d[v]) for v in range(V)])

    x = np.random.RandomState(order).randn(4, V)
    excl = (d.pad(), eos, d.unk())
    hyps = O.search(x, beam=10 ** 6, K=V, blank=blank, exclude=excl, lm_fn=lm_fn, lm_weight=lm_weight, word_score=word_score,
                    eos=eos)
    assert sorted(h[0] for h in hyps) == sorted(y for y in _enumerate(x, blank) if not set(y) & set(excl))
    for y, s, _ in hyps:
        ref = _ctc_logp(x, y, blank) + lm_weight * a.sentence_logp(sym(y)) + word_score * len(y)
        assert abs(s - ref) < 1e-10


def _lexicon_entries(d):
    """Multi-spelling words and homographs over the pieces a, b, c."""
    i = d.index
    return [("ab", (i("a"), i("b"))), ("a", (i("a"),)), ("b", (i("b"),)), ("bb", (i("b"), i("b"))), ("ba", (i("b"), i("a"))),
            ("c", (i("c"),)), ("see", (i("c"),)), ("abc", (i("a"), i("b"), i("c"))), ("ab", (i("a"), i("c"), i("b")))]


def _word_arpa(tmp_path, entries, order, seed):
    words = []
    for w, _ in entries:
        if w not in words:
            words.append(w)
    return N.write_arpa(tmp_path / "words.arpa", order, n_words=len(words), n_sent=150, seed=seed, words=words)


@pytest.mark.parametrize("T,order,lm_weight,word_score,seed", [(3, 2, 0.6, -0.4, 0), (4, 3, 1.1, 0.3, 1), (5, 2, 0.3, 0.0, 2)])
def test_lexicon_oracle_is_exhaustive(tmp_path, T, order, lm_weight, word_score, seed):
    d = _dict(n_sym=3)
    V, blank = len(d), 0
    entries = _lexicon_entries(d)
    a = _word_arpa(tmp_path, entries, order, seed)
    x = np.random.RandomState(seed).randn(T, V) * 1.5
    excl = (d.pad(), d.eos(), d.unk())
    hyps = N.search_lexicon(x, 10 ** 6, V, blank, entries, a, excl, math.inf, lm_weight, word_score)
    # every word sequence whose concatenated spellings form a reachable label sequence
    reach = {y for y in _enumerate(x, blank) if not set(y) & set(excl)}
    spell = {}
    for w, sp in entries:
        spell.setdefault(w, []).append(sp)
    words = list(spell)
    want = {}
    for n in range(0, T + 1):
        for ws in itertools.product(range(len(words)), repeat=n):
            for sps in itertools.product(*[spell[words[w]] for w in ws]):
                y = tuple(t for sp in sps for t in sp)
                if y in reach:
                    want.setdefault((y, ws), set()).add(sps)
    got = {(y, ws): s for y, s, _, ws in hyps}
    assert set(got) == set(want)
    for (y, ws), s in got.items():
        ref = _ctc_logp(x, y, blank) + lm_weight * a.sentence_logp([words[w] for w in ws]) + word_score * len(ws)
        assert abs(s - ref) < 1e-10, (y, ws)
    # homographs: one spelling, two hypotheses
    c = (d.index("c"),)
    if c in reach:
        assert {ws for (y, ws) in got if y == c} == {(words.index("c"),), (words.index("see"),)}


@pytest.fixture
def ngram_ops(monkeypatch):
    from espresso_b200 import ops
    from oracle import ctc_beam_ops, ctc_ngram_ops, ops_ref

    for mod in (ops_ref, ctc_beam_ops, ctc_ngram_ops):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                monkeypatch.setattr(ops, name, getattr(mod, name))


@pytest.mark.parametrize("with_lexicon", [False, True])
def test_host_search_over_ops_ref_matches_the_oracle(tmp_path, ngram_ops, with_lexicon):
    from espresso_b200.models import NgramLanguageModel
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict(n_sym=3)
    V = len(d)
    entries = _lexicon_entries(d)
    if with_lexicon:
        a = _word_arpa(tmp_path, entries, 3, seed=4)
        (tmp_path / "lexicon.txt").write_text("".join("%s\t%s\n" % (w, " ".join(d[t] for t in sp)) for w, sp in entries))
        path = tmp_path / "words.arpa"
    else:
        a = _sym_arpa(tmp_path, d, 3, seed=4)
        path = tmp_path / "sym.arpa"
    lm = NgramLanguageModel.from_arpa(str(path))
    beam, K, thr, lw, ws = 5, 4, 8.0, 0.9, -0.2
    dec = CTCDecoder(d, blank_idx=0, beam_size=beam, lm_model=lm, lm_weight=lw, word_score=ws, beam_size_token=K,
                     beam_threshold=thr, nbest=3, print_alignment=True,
                     lexicon=str(tmp_path / "lexicon.txt") if with_lexicon else None)
    B, T = 3, 8
    x = _logits(B, T, V, seed=9)
    lens = torch.tensor([8, 5, 0])
    tokens, lens_o, scores, frames = dec.search(x, V, lens)
    excl = (d.pad(), d.eos(), d.unk())
    for b in range(B):
        xb = x[b, : int(lens[b]), :V].double().numpy()
        if with_lexicon:
            ref = [r[:3] for r in N.search_lexicon(xb, beam, K, 0, entries, a, excl, thr, lw, ws)]
        else:
            lm_fn = lambda y: np.array([a.logp(["<s>"] + [d[v] for v in y], d[v]) for v in range(V)])  # noqa: E731
            ref = O.search(xb, beam, K, 0, excl, thr, lm_fn, lw, ws, d.eos())
        for r in range(3):
            if r >= len(ref):
                assert scores[b, r] == -math.inf
                continue
            y, s, fr = ref[r]
            n = int(lens_o[b, r])
            assert tuple(tokens[b, r, :n].tolist()) == y and (tokens[b, r, n:] == d.pad()).all()
            assert tuple(frames[b, r, :n].tolist()) == fr
            assert abs(float(scores[b, r]) - s) <= 1e-5 * max(1.0, abs(s))


def test_decoder_surface_and_refusals(tmp_path):
    from espresso_b200.models import NgramLanguageModel
    from espresso_b200.sequence_generator import SequenceGenerator
    from espresso_b200.tools.ctc_decoder import CTCDecoder
    from espresso_b200.tools.transducer_greedy_decoder import TransducerGreedyDecoder

    d = _dict(n_sym=3)
    lm = _load(tmp_path, TOY)
    assert isinstance(lm, NgramLanguageModel)
    dec = CTCDecoder(d, beam_size=1, lm_model=lm)
    assert not dec.greedy and dec.ngram and dec.lexicon is None
    assert dec._tok_word.tolist()[d.index("a")] == lm.index("a") and dec._tok_word.tolist()[d.eos()] == lm.eos
    with pytest.raises(NotImplementedError, match="KenLM.*NgramLanguageModel.from_arpa"):
        CTCDecoder(d, beam_size=4, lm_model=str(tmp_path / "lm.arpa"))
    (tmp_path / "lex.txt").write_text("ab a b\nzz a q\n")
    with pytest.raises(ValueError, match="missing from the dictionary"):
        CTCDecoder(d, beam_size=4, lm_model=lm, lexicon=str(tmp_path / "lex.txt"))
    with pytest.raises(NotImplementedError, match="n-gram LMs are fused into CTC decoding only"):
        SequenceGenerator([object()], d, beam_size=2, lm_model=lm, max_len=5)
    with pytest.raises(NotImplementedError, match="n-gram LMs are fused into CTC decoding only"):
        TransducerGreedyDecoder([object()], d, lm_model=lm)


def test_lexicon_trie_layout(tmp_path):
    from espresso_b200.models import LexiconTrie

    d = _dict(n_sym=3)
    entries = _lexicon_entries(d)
    lm = _load(tmp_path, TOY)
    t = LexiconTrie.build([[w] + [d[u] for u in sp] for w, sp in entries], d, lm)
    assert t.words == ["ab", "a", "b", "bb", "ba", "c", "see", "abc"]
    assert t.max_words == 2  # "c" and "see" share one spelling
    i = d.index

    def walk(sp):
        n = 0
        for u in sp:
            e0, e1 = t.child_off[n], t.child_off[n + 1]
            j = e0 + int(np.searchsorted(t.child_tok[e0:e1], u))
            assert j < e1 and t.child_tok[j] == u
            n = int(t.child_node[j])
        return n

    ends = lambda n: t.node_words[t.word_off[n]:t.word_off[n + 1]].tolist()  # noqa: E731
    assert ends(walk([i("c")])) == [5, 6] and ends(walk([i("a"), i("b")])) == [0] and ends(walk([i("a"), i("c"), i("b")])) == [0]
    assert t.word_lm.tolist() == [lm.index(w) for w in t.words]
    sm = t.compute_smear(np.arange(len(t.words), dtype=np.float64) * -1.0)
    assert sm[0] == 0.0 and sm[walk([i("a")])] == -0.0 and sm[walk([i("b")])] == -2.0 and sm[walk([i("a"), i("c")])] == -0.0


def test_build_generator_ctc_with_arpa_and_lexicon(tmp_path, ngram_ops):
    """build_generator on a CTC task routes an n-gram LM, `lexicon` and `word_score` (as recognize() hands them) to the
    decoder; every hypothesis it generates is a sequence of lexicon spellings."""
    from espresso_b200.models import NgramLanguageModel
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict(n_sym=3)
    V = len(d)
    task = _task(d)
    entries = _lexicon_entries(d)
    _word_arpa(tmp_path, entries, 2, seed=3)
    (tmp_path / "lexicon.txt").write_text("".join("%s %s\n" % (w, " ".join(d[t] for t in sp)) for w, sp in entries))
    lm = NgramLanguageModel.from_arpa(str(tmp_path / "words.arpa"))
    x = _logits(2, 7, V, seed=5, peaked=True)
    model = _FakeCTC(x, torch.tensor([7, 4]), V)
    g = task.build_generator([model], Namespace(beam=4, lm_weight=0.8, word_score=0.5, lexicon=str(tmp_path / "lexicon.txt"),
                                                nbest=2), extra_gen_cls_kwargs={"lm_model": lm, "lm_weight": 0.8})
    assert isinstance(g, CTCDecoder) and g.lexicon is not None and g.word_score == 0.5
    hy = g.generate([model], {"net_input": {}})
    spellings = {tuple(sp) for _, sp in entries}
    for hs in hy:
        for h in hs:
            y = tuple(h["tokens"].tolist())
            # a concatenation of lexicon spellings
            ok = {0}
            for p in range(1, len(y) + 1):
                if any(q in ok and y[q:p] in spellings for q in range(p)):
                    ok.add(p)
            assert len(y) in ok


def test_recognize_with_arpa_and_lexicon_scores_every_utterance(tmp_path, ngram_ops):
    """recognize() on a CTC task with an ARPA and a lexicon: utterances whose posteriors spell a whole lexicon word
    decode to it; an utterance that ends inside a word has no whole-word hypothesis, gets the empty one at score -inf,
    and is still written and scored (every word of its reference counts as deleted)."""
    import os

    from test_input_pipeline import _corpus

    from espresso_b200.data.asr_dictionary import AsrDictionary
    from espresso_b200.models import NgramLanguageModel
    from espresso_b200.speech_recognize import recognize
    from espresso_b200.tasks.speech_recognition import SpeechRecognitionEspressoConfig, SpeechRecognitionEspressoTask

    d0, man = _corpus(tmp_path, n=5, fmt="wave")
    os.rename(str(tmp_path / "train.json"), str(tmp_path / "test.json"))
    d = AsrDictionary(enable_bos=True)
    for s in d0.symbols[d0.nspecial:]:
        d.add_symbol(s)
    d.space_index = d.index("<space>")
    d.build_bpe("characters_asr")
    task = SpeechRecognitionEspressoTask(SpeechRecognitionEspressoConfig(criterion_name="ctc_loss", data=str(tmp_path)), d,
                                         feat_dim=80)
    (tmp_path / "lexicon.txt").write_text("ab a b\n")
    N.write_arpa(tmp_path / "w.arpa", 2, n_words=1, n_sent=20, seed=0, words=["ab"])
    lm = NgramLanguageModel.from_arpa(str(tmp_path / "w.arpa"))
    V, blank, a, b = len(d), d.bos(), d.index("a"), d.index("b")

    class Spelling(torch.nn.Module):
        """Posteriors that spell "a b" for even positions in the batch and only "a" (a cut word) for odd ones."""

        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.zeros(1))

        def forward(self, src_tokens, src_lengths, **unused):
            B, T = src_lengths.numel(), 12
            x = torch.full((B, T, (V + 7) // 8 * 8), -8.0)
            x[:, :, blank] = 8.0
            x[:, 0:3, blank] = -8.0
            x[:, 0:3, a] = 8.0
            x[0::2, 4:7, blank] = -8.0
            x[0::2, 4:7, b] = 8.0
            return {"b200_out": x.bfloat16(), "encoder_out": [torch.zeros(1, 1, V)],
                    "src_lengths": [torch.full((B,), T, dtype=torch.int32)]}

    out = recognize(task, [Spelling()], subset="test", gen_args=Namespace(beam=4, lm_weight=1.0, word_score=0.5,
                                                                          lexicon=str(tmp_path / "lexicon.txt")),
                    lms=[lm], max_tokens=None, max_sentences=2, device="cpu")
    h_lines = [l.split("\t") for l in out["lines"] if l.startswith("H-")]
    assert len(h_lines) == len(man) == out["num_sentences"]
    assert {l[1] for l in h_lines} == {"ab", ""}
    assert all((l[1] == "") == (float(l[2]) == -math.inf) for l in h_lines)
    assert len(out["scorer"].results) == len(man)  # every utterance reached the WER
