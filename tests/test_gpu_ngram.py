"""GPU: the n-gram LM kernels (esp_ngram_score, esp_ctc_ngram_search / _finalize) against oracle/ngram.py in float64.
Same rules as tests/test_gpu_ctc_beam.py: tokens exact wherever the oracle's score margin to the neighbouring ranks
exceeds MARGIN, scores within SCORE_TOL relative; each case records its error through the `parity` fixture."""
import math

import numpy as np
import pytest
import torch

from oracle import ctc_beam as O
from oracle import ngram as N
from oracle.ctc_ngram_ops import probe, state_of
from test_ctc_beam_search import _dict
from test_gpu_ctc_beam import MARGIN, SCORE_TOL, _repeat_heavy, _x

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.mark.parametrize("order", [2, 3, 4, 5, 6])
def test_ngram_score_matches_the_oracle(tmp_path, order, parity):
    from espresso_b200 import ops
    from espresso_b200.models import NgramLanguageModel

    a = N.write_arpa(tmp_path / "w.arpa.gz", order, n_words=60, n_sent=600, seed=order)
    lm = NgramLanguageModel.from_arpa(str(tmp_path / "w.arpa.gz"))
    rs = np.random.RandomState(order)
    words = a.vocab + ["oov"]
    n = 20000  # x 5 orders = 10^5 pairs
    hists = [["<s>"] + [words[i] for i in rs.randint(0, len(words), size=rs.randint(0, order + 1))] for _ in range(n)]
    ws = [words[i] for i in rs.randint(0, len(words), size=n)]
    cache = {}
    st = []
    for h in hists:
        key = tuple(h)
        if key not in cache:
            cache[key] = state_of(lm, [lm.index(x) for x in h[1:]])
        st.append(cache[key])
    wid = [lm.index(w) for w in ws]
    lp, nxt = ops.ngram_score(lm, torch.tensor(st, dtype=torch.int32, device=DEV), torch.tensor(wid, dtype=torch.int32, device=DEV))
    lp, nxt = lp.cpu().numpy(), nxt.cpu().numpy()
    err = 0.0
    for i in range(n):
        ref = a.logp(hists[i], ws[i])
        err = max(err, abs(float(lp[i]) - ref) / max(1.0, abs(ref)))
        if i < 2000:
            assert int(nxt[i]) == probe(lm, st[i], wid[i])[1]
    parity("esp_ngram_score order %d: log10 rel err" % order, err, 1e-6)


# ---- searches -------------------------------------------------------------------------------------------------------
def _check(parity, name, got, refs, nbest, check):
    """got = CTCDecoder.search output; refs[b] = the oracle's (tokens, score, frames) list of sentence b."""
    tokens, L, S, Fr = got
    err, n_exact = 0.0, 0  # ranks checked against the oracle
    for b in check:
        ref = refs[b]
        sc = [r[1] for r in ref]
        for r in range(nbest):
            if r >= len(ref):
                assert S[b, r] == -math.inf
                continue
            gap = min(sc[r - 1] - sc[r] if r > 0 else math.inf, sc[r] - sc[r + 1] if r + 1 < len(sc) else math.inf)
            m = int(L[b, r])
            got_y = tuple(tokens[b, r, :m].tolist())
            if gap > MARGIN:
                assert got_y == ref[r][0], (name, b, r)
                err = max(err, abs(float(S[b, r]) - sc[r]) / max(1.0, abs(sc[r])))
                if Fr is not None:
                    assert tuple(Fr[b, r, :m].tolist()) == ref[r][2]
                n_exact += 1
            else:  # a near-tie (homographs tie exactly) may swap ranks: the hypothesis must be one of the oracle's
                alt = [h for h in ref if h[0] == got_y]
                if alt:
                    err = max(err, min(abs(float(S[b, r]) - h[1]) for h in alt) / max(1.0, abs(alt[0][1])))
                    n_exact += 1
    assert n_exact > 0
    parity(name + ": score rel err", err, SCORE_TOL)


def _sym_lm(tmp_path, d, order, seed):
    from espresso_b200.models import NgramLanguageModel

    pieces = [d[i] for i in range(d.nspecial, len(d))]
    a = N.write_arpa(tmp_path / "sym.arpa", order, n_words=len(pieces), n_sent=400, seed=seed, words=pieces)
    return a, NgramLanguageModel.from_arpa(str(tmp_path / "sym.arpa"))


def _free_refs(x, lens, dec, a, d, V, K, thr, check):
    excl = (dec.pad, dec.eos, dec.unk)
    syms = [d[v] for v in range(V)]
    refs = {}
    for b in check:
        cache = {}

        def lm_fn(y):
            if y not in cache:
                cache[y] = a.logp_vector(["<s>"] + [d[v] for v in y], syms)
            return cache[y]

        refs[b] = O.search(x[b, : int(lens[b]), :V].double().numpy(), dec.beam_size, K, dec.blank, excl, thr, lm_fn,
                           dec.lm_weight, dec.word_score, dec.eos)
    return refs


@pytest.mark.parametrize("beam,order,case", [(4, 2, "random"), (16, 3, "repeat"), (60, 4, "random")])
def test_lexicon_free_search(tmp_path, beam, order, case, parity):
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    V, B, T = 28, 4, 40
    d = _dict(n_sym=V - 4)
    a, lm = _sym_lm(tmp_path, d, order, seed=beam)
    x = _x(B, T, V, seed=beam, scale=2.0) if case == "random" else _repeat_heavy(B, T, V, seed=beam)
    lens = torch.tensor([40, 23, 1, 0])
    dec = CTCDecoder(d, blank_idx=0, beam_size=beam, lm_model=lm, lm_weight=0.9, word_score=0.4, nbest=3, print_alignment=True)
    got = dec.search(x.to(DEV), V, lens.to(DEV))
    K, thr = min(beam, V), float(min(beam, V))
    _check(parity, "ctc + %d-gram lexicon-free beam=%d %s" % (order, beam, case), got,
           _free_refs(x, lens, dec, a, d, V, K, thr, range(B)), 3, range(B))


def _lexicon(d, n_words, seed, min_len=1, max_len=3):
    """Random spellings over the dictionary's pieces; every 7th word gets a second spelling and every 11th shares the
    spelling of the word before it (a homograph)."""
    rs = np.random.RandomState(seed)
    pieces = list(range(d.nspecial, len(d)))
    entries = []
    for i in range(n_words):
        w = "w%d" % i
        sp = tuple(int(p) for p in rs.choice(pieces, size=rs.randint(min_len, max_len + 1)))
        if i % 11 == 10:
            sp = entries[-1][1]
        entries.append((w, sp))
        if i % 7 == 6:
            entries.append((w, tuple(int(p) for p in rs.choice(pieces, size=rs.randint(min_len, max_len + 1)))))
    return entries


def _lex_decoder(tmp_path, d, entries, order, seed, beam, **kw):
    from espresso_b200.models import NgramLanguageModel
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    words = list(dict.fromkeys(w for w, _ in entries))
    a = N.write_arpa(tmp_path / "words.arpa", order, n_words=len(words), n_sent=kw.pop("n_sent", 400), seed=seed, words=words)
    (tmp_path / "lexicon.txt").write_text("".join("%s\t%s\n" % (w, " ".join(d[t] for t in sp)) for w, sp in entries))
    lm = NgramLanguageModel.from_arpa(str(tmp_path / "words.arpa"))
    dec = CTCDecoder(d, blank_idx=0, beam_size=beam, lm_model=lm, lexicon=str(tmp_path / "lexicon.txt"), **kw)
    return a, dec


def _lex_refs(x, lens, dec, a, entries, V, K, thr, check):
    excl = (dec.pad, dec.eos, dec.unk)
    return {b: [r[:3] for r in N.search_lexicon(x[b, : int(lens[b]), :V].double().numpy(), dec.beam_size, K, dec.blank, entries,
                                                  a, excl, thr, dec.lm_weight, dec.word_score)] for b in check}


@pytest.mark.parametrize("beam,order,case", [(4, 2, "random"), (16, 3, "repeat"), (40, 3, "random")])
def test_lexicon_search(tmp_path, beam, order, case, parity):
    V, B, T = 20, 4, 36
    d = _dict(n_sym=V - 4)
    entries = _lexicon(d, 40, seed=beam)
    a, dec = _lex_decoder(tmp_path, d, entries, order, beam, beam, lm_weight=0.8, word_score=-0.3, nbest=3, print_alignment=True)
    assert dec.lexicon.max_words >= 2
    x = _x(B, T, V, seed=beam, scale=2.0) if case == "random" else _repeat_heavy(B, T, V, seed=beam)
    lens = torch.tensor([36, 20, 1, 0])
    got = dec.search(x.to(DEV), V, lens.to(DEV))
    K, thr = min(beam, V), float(min(beam, V))
    _check(parity, "ctc + %d-gram lexicon beam=%d %s" % (order, beam, case), got, _lex_refs(x, lens, dec, a, entries, V, K, thr,
                                                                                           range(B)), 3, range(B))


def _spelled(lens, T, V, entries, seed, peak=12.0):
    """Noise plus peaks that spell random lexicon words, one to three frames per unit with blanks between some of them,
    up to the last whole word that fits each sentence, then blanks (a trained model's posteriors on in-lexicon speech)."""
    rs = np.random.RandomState(seed)
    x = rs.randn(len(lens), T, (V + 7) // 8 * 8)
    for b, n in enumerate(lens.tolist()):
        t = 0
        while True:
            plan = [(u, rs.randint(1, 4)) for v in entries[rs.randint(len(entries))][1]
                    for u in ([0] if rs.rand() < 0.4 else []) + [v]]
            if t + sum(k for _, k in plan) > n:
                break
            for u, k in plan:
                x[b, t:t + k, u] += peak
                t += k
        x[b, t:, 0] += peak
    return torch.from_numpy(x).float().bfloat16()


@pytest.mark.parametrize("beam", [10, 60])
def test_recipe_shape(tmp_path, beam, parity):
    """V = 5004 pieces, 24 x 250 frames, K = beam, a 3-gram over 20 000 words and a lexicon with multi-spelling words
    and homographs; one launch for the search, both modes; the oracle checks a subset of the sentences."""
    from espresso_b200 import lib

    V, B, T = 5004, 24, 250
    d = _dict(n_sym=V - 4)
    entries = _lexicon(d, 20000, seed=1, min_len=2, max_len=4)
    a, dec = _lex_decoder(tmp_path, d, entries, 3, 1, beam, lm_weight=1.0, word_score=0.5, nbest=2, n_sent=4000)
    lens = torch.tensor([T - 7 * b for b in range(B)])
    x = _spelled(lens, T, V, entries, seed=beam)
    check = [0, 13] if beam == 10 else [5]
    dec.search(x.to(DEV), V, lens.to(DEV))  # the first call uploads the tables and smears the trie
    c0 = lib.launch_count()
    got = dec.search(x.to(DEV), V, lens.to(DEV))
    assert lib.launch_count() - c0 == 3  # frames, one search launch for all frames, finalize
    _check(parity, "ctc + 3-gram lexicon recipe shape beam=%d" % beam, got, _lex_refs(x, lens, dec, a, entries, V, beam,
                                                                                     float(beam), check), 2, check)
    a2, lm2 = _sym_lm(tmp_path, d, 3, seed=beam)
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    dec2 = CTCDecoder(d, blank_idx=0, beam_size=beam, lm_model=lm2, lm_weight=0.6, word_score=0.2, nbest=2)
    dec2.search(x.to(DEV), V, lens.to(DEV))
    c0 = lib.launch_count()
    got = dec2.search(x.to(DEV), V, lens.to(DEV))
    assert lib.launch_count() - c0 == 3
    _check(parity, "ctc + 3-gram lexicon-free recipe shape beam=%d" % beam, got,
           _free_refs(x, lens, dec2, a2, d, V, beam, float(beam), check[:1]), 2, check[:1])


def test_capacity_is_refused():
    from espresso_b200 import lib, ops
    from espresso_b200.models import LexiconTrie

    V = 20
    d = _dict(n_sym=V - 4)
    lm = None
    import tempfile

    with tempfile.TemporaryDirectory() as tmp:
        N.write_arpa(tmp + "/w.arpa", 2, n_words=5, n_sent=20, seed=0, words=["a", "b", "c", "d", "e"])
        from espresso_b200.models import NgramLanguageModel

        lm = NgramLanguageModel.from_arpa(tmp + "/w.arpa")
    trie = LexiconTrie.build([[w, "a"] for w in ("a", "b", "c", "d", "e")], d, lm)  # five homographs
    x = _x(1, 4, V, seed=0).to(DEV)
    lens = torch.tensor([4], dtype=torch.int32, device=DEV)
    fr = ops.ctc_beam_frames(x, V, lens, 128, 0)
    ws = ops.ctc_ngram_workspace(1, 4, 128, DEV)
    with pytest.raises(lib.EspressoB200Error, match="does not fit in shared memory"):
        ops.ctc_ngram_search(x, V, lens, fr, 128, 10.0, ws, lm, lexicon=trie)
    ops.ctc_ngram_search(x, V, lens, ops.ctc_beam_frames(x, V, lens, 16, 0), 16, 10.0, ws, lm, lexicon=trie)
    torch.cuda.synchronize()


def test_token_map_narrower_than_the_logits_is_refused(tmp_path):
    """Lexicon-free, every top-K token indexes the token -> word map: logits wider than the dictionary are refused."""
    from espresso_b200 import lib, ops

    V = 24
    d = _dict(n_sym=V - 4)
    _, lm = _sym_lm(tmp_path, d, 2, seed=0)
    x = _x(1, 6, V + 8, seed=0).to(DEV)
    lens = torch.tensor([6], dtype=torch.int32, device=DEV)
    tw = torch.tensor([lm.index(d[i]) for i in range(V)], dtype=torch.int32, device=DEV)
    ws = ops.ctc_ngram_workspace(1, 6, 4, DEV)
    with pytest.raises(lib.EspressoB200Error, match="tok_word maps 24 tokens, the CTC vocabulary has 32"):
        ops.ctc_ngram_search(x, V + 8, lens, ops.ctc_beam_frames(x, V + 8, lens, 4, 0), 4, 4.0, ws, lm, tok_word=tw)
    ops.ctc_ngram_search(x, V, lens, ops.ctc_beam_frames(x, V, lens, 4, 0), 4, 4.0, ws, lm, tok_word=tw)
    torch.cuda.synchronize()


def test_fixture_conformer_with_arpa(tmp_path, golden_dir, parity):
    import os

    from espresso_b200.tools.ctc_decoder import CTCDecoder
    from test_gpu_encoder import _build, _sample

    g = np.load(os.path.join(golden_dir, "encoder_conformer.npz"))
    m = _build("conformer", g)
    m.eval()
    sample = _sample(g, DEV)
    with torch.no_grad():
        net = m(**sample["net_input"])
    V = net["encoder_out"][0].size(-1)
    x = net["b200_out"].cpu()
    lens = net["src_lengths"][0].cpu()
    d = _dict(n_sym=V - 4)
    a, lm = _sym_lm(tmp_path, d, 3, seed=2)
    dec = CTCDecoder(d, blank_idx=0, beam_size=8, lm_model=lm, lm_weight=0.5, word_score=0.2, nbest=2)
    got = dec.search(x.to(DEV), V, lens.to(DEV))
    _check(parity, "ctc + 3-gram fixture conformer", got, _free_refs(x, lens, dec, a, d, V, 8, 8.0, range(x.shape[0])), 2,
           range(x.shape[0]))
    tok, sc, _ = dec.decode([m], sample)
    hy = dec.generate([m], sample)
    for b, h in enumerate(hy):
        assert torch.equal(h[0]["tokens"], tok[b, : h[0]["tokens"].numel()]) and h[0]["score"] == float(sc[b])
