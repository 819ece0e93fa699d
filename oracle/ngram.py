"""Oracle: ARPA n-gram language models and CTC prefix beam search through a word lexicon, in float64 numpy / Python.

TEST INFRASTRUCTURE ONLY; imports nothing from espresso_b200.  Three pieces:
  Arpa        an ARPA reader and scorer written straight from the backoff recursion over full word histories (no
              states): log10 P(w | h) = prob(h w) if listed, else backoff(h) (0 when h is not listed) + log10 P(w | h
              without its first word); at the empty history the 1-gram of w (of <unk> for an unknown word; an ARPA
              without <unk> gives it -100, as KenLM does).  Histories are cut to the last order - 1 words.
  write_arpa  a seeded writer: a Zipf corpus, add-one 1-grams, absolute discounting above them, and backoff weights
              normalised so that sum_w P(w | h) = 1 for every history.
  search_lexicon / lexicon_step / lexicon_finish
              the statement of espresso_b200/csrc/ctc_beam.cu's lexicon mode (oracle/ctc_beam.py's search, plus):
                a hypothesis also holds its trie position (the spelling units since its last word), its completed
                words with their positions (its segmentation) and a look-ahead term; score = lae(pb, pnb) + lm + la;
                extending with v needs the position + (v,) to prefix a spelling; per (slot, token rank) the candidates
                are the in-word continuation (when a longer spelling continues, la = lm_weight * smear) and then the
                words spelled exactly so, by ascending word id (lm += lm_weight * log10 P(w | words) + word_score,
                la = 0, back to the root); candidate index h * (1 + K * W1) + 1 + rank * W1 + q, W1 = 1 + the most
                words sharing one spelling; candidates merge only when tokens and segmentation agree;
                finish keeps hypotheses at the root, + lm_weight * log10 P(</s> | words).
              smear(position) = max over the words whose spelling starts with it of log10 P(w | <s>); 0 at the root."""
import gzip
import math
from collections import Counter, namedtuple

import numpy as np

from oracle import ctc_beam as O

NEG = -math.inf


class Arpa:
    def __init__(self, order, grams):
        self.order, self.grams = order, grams  # grams[k - 1][(w1, .., wk)] = (log10 prob, log10 backoff)
        if ("<unk>",) not in grams[0]:
            grams[0][("<unk>",)] = (-100.0, 0.0)
        self.vocab = [g[0] for g in grams[0]]

    @classmethod
    def read(cls, path):
        opener = gzip.open if str(path).endswith(".gz") else open
        with opener(path, "rt", encoding="utf-8") as f:
            lines = [l.strip() for l in f]
        i = lines.index("\\data\\") + 1
        counts = []
        while lines[i].startswith("ngram "):
            counts.append(int(lines[i].split("=")[1]))
            i += 1
        grams = []
        for k in range(1, len(counts) + 1):
            i = lines.index("\\%d-grams:" % k, i) + 1
            g = {}
            while lines[i] and not lines[i].startswith("\\"):
                f = lines[i].split()
                g[tuple(f[1:k + 1])] = (float(f[0]), float(f[k + 1]) if len(f) > k + 1 else 0.0)
                i += 1
            assert len(g) == counts[k - 1]
            grams.append(g)
        return cls(len(counts), grams)

    def _known(self, w):
        return w if (w,) in self.grams[0] else "<unk>"

    def logp(self, hist, w):
        """log10 P(w | hist), hist a sequence of words (starting with "<s>" for a sentence)."""
        h = tuple(self._known(x) for x in hist)
        h = h[max(0, len(h) - (self.order - 1)):] if self.order > 1 else ()
        return self._p(h, self._known(w))

    def _p(self, h, w):
        if not h:
            return self.grams[0][(w,)][0]
        g = self.grams[len(h)].get(h + (w,))
        if g is not None:
            return g[0]
        return self.grams[len(h) - 1].get(h, (0.0, 0.0))[1] + self._p(h[1:], w)

    def logp_vector(self, hist, words):
        """[log10 P(w | hist) for w in words], the same recursion run for all words at once."""
        if not hasattr(self, "_children"):
            self._children = {}
            for k in range(1, self.order):
                for g, (p, _) in self.grams[k].items():
                    self._children.setdefault(g[:-1], []).append((g[-1], p))
        known = [self._known(w) for w in words]
        pos = {}
        for i, w in enumerate(known):
            pos.setdefault(w, []).append(i)
        v = np.array([self.grams[0][(w,)][0] for w in known], dtype=np.float64)
        h = tuple(self._known(x) for x in hist)
        h = h[max(0, len(h) - (self.order - 1)):] if self.order > 1 else ()
        for k in range(1, len(h) + 1):
            ctx = h[len(h) - k:]
            v = v + self.grams[k - 1].get(ctx, (0.0, 0.0))[1]
            for w, p in self._children.get(ctx, ()):
                for i in pos.get(w, ()):
                    v[i] = p
        return v

    def sentence_logp(self, words):
        ctx, s = ["<s>"], 0.0
        for w in list(words) + ["</s>"]:
            s += self.logp(ctx, w)
            ctx.append(w)
        return s


def zipf_corpus(n_words, n_sent, seed, max_len=12, words=None):
    rs = np.random.RandomState(seed)
    words = words or ["w%d" % i for i in range(n_words)]
    p = 1.0 / np.arange(1, n_words + 1)
    p /= p.sum()
    return words, [[words[i] for i in rs.choice(n_words, size=rs.randint(1, max_len + 1), p=p)] for _ in range(n_sent)]


def write_arpa(path, order, n_words=30, n_sent=300, seed=0, discount=0.7, with_unk=True, words=None):
    """A normalised backoff model of `order` from a seeded Zipf corpus over n_words words (w0, w1, .. unless `words`),
    written as ARPA (gzip when path ends in .gz).  Returns the Arpa."""
    words, sents = zipf_corpus(n_words, n_sent, seed, words=words)
    counts = [Counter() for _ in range(order)]
    for s in sents:
        toks = ["<s>"] + s + ["</s>"]
        for k in range(1, order + 1):
            for i in range(len(toks) - k + 1):
                g = tuple(toks[i:i + k])
                if k == 1 and g == ("<s>",):
                    continue
                counts[k - 1][g] += 1
    vocab = ["</s>"] + (["<unk>"] if with_unk else []) + list(words)
    total = sum(counts[0][(w,)] for w in vocab)
    grams = [{("<s>",): (-99.0, 0.0)}]
    for w in vocab:
        grams[0][(w,)] = (math.log10((counts[0][(w,)] + 1) / (total + len(vocab))), 0.0)
    for k in range(2, order + 1):
        ctx_total, ctx_types = Counter(), Counter()
        for g, c in counts[k - 1].items():
            ctx_total[g[:-1]] += c
            ctx_types[g[:-1]] += 1
        grams.append({g: (math.log10((c - discount) / ctx_total[g[:-1]]), 0.0) for g, c in counts[k - 1].items()})
        # backoff weights of the (k-1)-grams, against the model of order k - 1
        lower = Arpa(k - 1, [dict(x) for x in grams[:k - 1]])
        seen = {}
        for g in grams[k - 1]:
            seen.setdefault(g[:-1], []).append(g[-1])
        for h, p in list(grams[k - 2].items()):
            if h not in seen:
                continue
            alpha = discount * ctx_types[h] / ctx_total[h]
            covered = sum(10.0 ** lower._p(h[1:], w) for w in seen[h])
            grams[k - 2][h] = (p[0], math.log10(alpha / (1.0 - covered)))
    opener = gzip.open if str(path).endswith(".gz") else open
    with opener(path, "wt", encoding="utf-8") as f:
        f.write("\\data\\\n")
        for k in range(order):
            f.write("ngram %d=%d\n" % (k + 1, len(grams[k])))
        for k in range(order):
            f.write("\n\\%d-grams:\n" % (k + 1))
            for g, (p, bo) in grams[k].items():
                f.write("%r\t%s" % (p, " ".join(g)) + ("\t%r\n" % bo if k + 1 < order else "\n"))
        f.write("\n\\end\\\n")
    return Arpa.read(path)


# ---- CTC prefix beam search through a word lexicon --------------------------------------------------------------------
class Lexicon:
    """entries: [(word, spelling tuple of CTC units)]; word ids by first appearance."""

    def __init__(self, entries, start_logp):
        self.words, wid = [], {}
        self.ends = {}
        for w, sp in entries:
            if w not in wid:
                wid[w] = len(self.words)
                self.words.append(w)
            self.ends.setdefault(tuple(sp), set()).add(wid[w])
        self.ends = {k: sorted(v) for k, v in self.ends.items()}
        self.prefixes = {sp[:i] for sp in self.ends for i in range(1, len(sp) + 1)}
        self.inner = {sp[:i] for sp in self.ends for i in range(1, len(sp))}  # positions a longer spelling continues
        self.max_words = max(len(v) for v in self.ends.values())
        self.smear = {(): 0.0}
        for sp, ws in self.ends.items():
            best = max(start_logp(w) for w in ws)
            for i in range(1, len(sp) + 1):
                self.smear[sp[:i]] = max(self.smear.get(sp[:i], NEG), best)


LHyp = namedtuple("LHyp", "y pb pnb lm la node words seg frames")


def lexicon_initial(dt=np.float64):
    return [LHyp((), dt(0.0), dt(NEG), dt(0.0), dt(0.0), (), (), (), ())]


def lexicon_step(hyps, t, lp, lp_blank, tok, beam, threshold, lex, lm_fn, lm_weight, word_score, dt=np.float64):
    """One frame; lm_fn(word ids tuple, word id) -> log10 P.  Returns (new hypotheses in slot order, sources)."""
    lae = lambda a, b: dt(np.logaddexp(dt(a), dt(b)))  # noqa: E731
    K, W1 = len(tok), 1 + lex.max_words
    S1 = 1 + K * W1
    index = {(h.y, h.seg): i for i, h in enumerate(hyps)}
    lp = np.asarray(lp, dtype=dt)
    spb = [dt(lae(h.pb, h.pnb) + dt(lp_blank)) for h in hyps]
    spnb = [dt(h.pnb + lp[h.y[-1]]) if h.y else dt(NEG) for h in hyps]
    lw, ws = dt(lm_weight), dt(word_score)
    merge, cands = {}, []
    for i, h in enumerate(hyps):
        for r, v in enumerate(tok):
            v = int(v)
            c = h.node + (v,)
            if v < 0 or c not in lex.prefixes:
                continue
            e = dt((h.pb if (h.y and v == h.y[-1]) else lae(h.pb, h.pnb)) + lp[v])
            y2 = h.y + (v,)
            base = i * S1 + 1 + r * W1
            if c in lex.inner:
                if (y2, h.seg) in index:
                    merge[index[(y2, h.seg)]] = e
                else:
                    la = dt(lw * dt(lex.smear[c]))
                    cands.append((dt(dt(e + h.lm) + la), base, LHyp(y2, dt(NEG), e, h.lm, la, c, h.words, h.seg,
                                                                   h.frames + (t,)), i, v))
            for q, w in enumerate(lex.ends.get(c, ()), 1):
                seg = h.seg + ((len(y2), w),)
                if (y2, seg) in index:
                    merge[index[(y2, seg)]] = e
                    continue
                lm = dt(dt(h.lm + ws) + dt(lw * dt(lm_fn(h.words, w))))
                cands.append((dt(dt(e + lm) + dt(0.0)), base + q, LHyp(y2, dt(NEG), e, lm, dt(0.0), (), h.words + (w,), seg,
                                                                      h.frames + (t,)), i, v))
    for i, h in enumerate(hyps):
        pnb = lae(spnb[i], merge.get(i, dt(NEG)))
        cands.append((dt(dt(lae(spb[i], pnb) + h.lm) + h.la), i * S1, h._replace(pb=spb[i], pnb=pnb), i, -1))
    cands = [c for c in cands if c[0] > NEG and not np.isnan(c[0])]
    if not cands:
        return [], []
    floor_ = dt(max(c[0] for c in cands) - dt(threshold))
    cands = sorted((c for c in cands if not c[0] < floor_), key=lambda c: (-c[0], c[1]))[:beam]
    return [c[2] for c in cands], [(c[3], c[4]) for c in cands]


def lexicon_finish(hyps, lm_fn, lm_weight, eos_word, dt=np.float64):
    """-> [(tokens, score, frames, words)] of the hypotheses at the root, by (score desc, slot asc)."""
    out = []
    for k, h in enumerate(hyps):
        if h.node:
            continue
        s = dt(dt(np.logaddexp(dt(h.pb), dt(h.pnb)) + h.lm) + h.la)
        s = dt(s + dt(dt(lm_weight) * dt(lm_fn(h.words, eos_word))))
        out.append((s, k, h))
    out.sort(key=lambda c: (-c[0], c[1]))
    return [(c[2].y, float(c[0]), c[2].frames, c[2].words) for c in out]


def arpa_word_fn(arpa, words):
    """lm_fn over lexicon word ids from an Arpa (float64 full-history recursion); word id -1 stands for </s>."""
    cache = {}

    def fn(hist, w):
        key = (hist, w)
        if key not in cache:
            cache[key] = arpa.logp(["<s>"] + [words[x] for x in hist], "</s>" if w < 0 else words[w])
        return cache[key]

    return fn


def search_lexicon(logits, beam, K, blank, entries, arpa, exclude=(), threshold=math.inf, lm_weight=0.0, word_score=0.0):
    """logits [T, V]; entries [(word, spelling)] -> every final hypothesis as (tokens, score, frames, word ids)."""
    x = np.asarray(logits, dtype=np.float64)
    lps = O.log_softmax(x)
    toks = O.topk_tokens(x, K, blank, exclude)
    words = []
    for w, _ in entries:
        if w not in words:
            words.append(w)
    lex = Lexicon(entries, lambda w: arpa.logp(["<s>"], words[w]))
    fn = arpa_word_fn(arpa, lex.words)
    hyps = lexicon_initial()
    for t in range(x.shape[0]):
        hyps, _ = lexicon_step(hyps, t, lps[t], lps[t, blank], toks[t], beam, threshold, lex, fn, lm_weight, word_score)
    return lexicon_finish(hyps, fn, lm_weight, -1)
