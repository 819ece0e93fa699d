"""ARPA n-gram language models for CTC decoding (the KenLM model of espresso/tools/ctc_decoder.py:22-73).

NgramLanguageModel.from_arpa(path) reads a .arpa or .arpa.gz file of order 1 to 6 through the host parser behind
esp_ngram_build (include/espresso_b200.h: the table layout and the scoring rule).  Scores are log10, KenLM's unit.
The tables are uploaded once per device and cached, like TensorizedPrefixTree.to.

LexiconTrie is flashlight's lexicon (a word, then its spelling in dictionary units, one spelling per line) as a trie in
the CSR edge layout of tools/tensorized_prefix_tree.py, with the words ending at each node and each node's smeared
look-ahead score, max over the words below it of log10 P(w | <s>) (0 at the root)."""
import ctypes as C
import gzip

import numpy as np
import torch

from .. import lib as _lib
from ..tools.tensorized_prefix_tree import csr_edges


class NgramLanguageModel:
    """Word ids follow the order of the ARPA's 1-grams (an added <unk> comes last)."""

    def __init__(self, order, counts, tables, vocab, start, eos, unk, unk_added):
        self.order, self.counts = order, list(counts)
        self.word, self.prob, self.backoff = tables["word"], tables["prob"], tables["backoff"]
        self.child_lo, self.child_hi, self.suffix = tables["child_lo"], tables["child_hi"], tables["suffix"]
        self.vocab = vocab
        self.indices = {w: i for i, w in enumerate(vocab)}
        self.start, self.eos, self.unk, self.unk_added = start, eos, unk, unk_added
        self.order_off = np.concatenate([[0], np.cumsum(self.counts)]).astype(np.int64)
        self._dev = {}

    @classmethod
    def from_arpa(cls, path):
        with open(path, "rb") as f:
            text = f.read()
        if text[:2] == b"\x1f\x8b":
            text = gzip.decompress(text)
        lib = _lib.load()
        t = _lib.EspArpaTables()
        _lib.check(lib.esp_ngram_build(text, len(text), C.byref(t)))
        counts = [int(t.count[k]) for k in range(t.order)]
        n = sum(counts)
        tables = {k: np.zeros(max(n, 1), dtype=np.float32 if k in ("prob", "backoff") else np.int32)
                  for k in ("word", "prob", "backoff", "child_lo", "child_hi", "suffix")}
        vocab = C.create_string_buffer(int(t.vocab_bytes))
        for k, a in tables.items():
            setattr(t, k, a.ctypes.data)
        t.vocab = C.cast(vocab, C.c_void_p)
        _lib.check(lib.esp_ngram_build(text, len(text), C.byref(t)))
        words = [w.decode("utf-8") for w in vocab.raw[:-1].split(b"\0")] if t.vocab_bytes else []
        assert len(words) == counts[0]
        return cls(t.order, counts, {k: a[:n] for k, a in tables.items()}, words, t.start, t.eos, t.unk, bool(t.unk_added))

    def index(self, word):
        """Word id, or <unk>'s for a word outside the 1-grams."""
        return self.indices.get(word, self.unk)

    def eval(self):
        return self

    @property
    def table_bytes(self):
        return sum(getattr(self, k).nbytes for k in ("word", "prob", "backoff", "child_lo", "child_hi", "suffix"))

    def to(self, device):
        """Device tables, cached per device: {name: tensor, "struct": EspNgram pointing at them}."""
        key = str(device)
        if key not in self._dev:
            d = {k: torch.from_numpy(np.ascontiguousarray(getattr(self, k))).to(device)
                 for k in ("word", "prob", "backoff", "child_lo", "child_hi", "suffix")}
            s = _lib.EspNgram()
            for k, v in d.items():
                setattr(s, k, v.data_ptr())
            s.order = self.order
            for i in range(7):
                s.order_off[i] = int(self.order_off[min(i, self.order)])
            s.start, s.eos, s.unk = self.start, self.eos, self.unk
            d["struct"] = s
            self._dev[key] = d
        return self._dev[key]


class LexiconTrie:
    """Node 0 is the root.  Word ids follow the lexicon's order of first appearance."""

    def __init__(self, words, child_off, child_tok, child_node, word_off, node_words, word_lm):
        self.words = words
        self.child_off, self.child_tok, self.child_node = child_off, child_tok, child_node
        self.word_off, self.node_words, self.word_lm = word_off, node_words, word_lm
        self.smear = None
        self._dev = {}

    @property
    def num_nodes(self):
        return len(self.word_off) - 1

    @property
    def max_words(self):
        return int(np.diff(self.word_off).max()) if self.num_nodes else 0

    @classmethod
    def from_file(cls, path, dictionary, lm):
        with open(path, encoding="utf-8") as f:
            return cls.build([line.split() for line in f if line.strip()], dictionary, lm)

    @classmethod
    def build(cls, entries, dictionary, lm):
        """entries: [word, unit, unit, ...] per spelling.  A unit outside `dictionary` raises ValueError."""
        words, wid, edge, ends = [], {}, {}, {}
        n = 1
        for e in entries:
            w, spell = e[0], e[1:]
            if not spell:
                raise ValueError("lexicon word %r has an empty spelling" % w)
            missing = [u for u in spell if u not in dictionary]
            if missing:
                raise ValueError("lexicon word %r is spelled with units missing from the dictionary: %s" % (w, missing))
            if w not in wid:
                wid[w] = len(words)
                words.append(w)
            node = 0
            for u in spell:
                key = (node, dictionary.index(u))
                if key not in edge:
                    edge[key] = n
                    n += 1
                node = edge[key]
            ends.setdefault(node, set()).add(wid[w])
        child_off, child_tok, child_node = csr_edges(edge, n)
        cnt = np.zeros(n + 1, dtype=np.int64)
        for node, ws in ends.items():
            cnt[node + 1] = len(ws)
        word_off = np.cumsum(cnt).astype(np.int32)
        node_words = np.zeros(int(word_off[-1]), dtype=np.int32)
        for node, ws in ends.items():
            node_words[word_off[node]:word_off[node + 1]] = sorted(ws)
        word_lm = np.array([lm.index(w) for w in words], dtype=np.int32)
        return cls(words, child_off, child_tok, child_node, word_off, node_words, word_lm)

    def compute_smear(self, logp_start):
        """smear[n] = max over the words below n of logp_start[word] (log10 P(w | <s>)), smear[root] = 0."""
        n = self.num_nodes
        sm = np.full(n, -np.inf, dtype=np.float64)
        node_of = np.repeat(np.arange(n), np.diff(self.word_off))
        np.maximum.at(sm, node_of, np.asarray(logp_start, dtype=np.float64)[self.node_words])
        parent = np.zeros(n, dtype=np.int64)
        parent[self.child_node] = np.repeat(np.arange(n), np.diff(self.child_off))
        for v in range(n - 1, 0, -1):  # a child's id is above its parent's
            if sm[v] > sm[parent[v]]:
                sm[parent[v]] = sm[v]
        sm[0] = 0.0
        return sm.astype(np.float32)

    def to(self, device, lm):
        """Device arrays, cached per device: {name: tensor, "struct": EspLexicon}.  The smear scores come from
        esp_ngram_score on the device."""
        from .. import ops

        key = str(device)
        if key not in self._dev:
            if self.smear is None:
                words = torch.from_numpy(self.word_lm).to(device)
                states = torch.full_like(words, lm.start)
                lp, _ = ops.ngram_score(lm, states, words)
                self.smear = self.compute_smear(lp.cpu().numpy())
            d = {}
            for k in ("child_off", "child_tok", "child_node", "word_off", "node_words", "word_lm", "smear"):
                a = getattr(self, k)
                d[k] = torch.from_numpy(np.ascontiguousarray(a if a.size else np.zeros(1, a.dtype))).to(device)
            s = _lib.EspLexicon()
            for k, f in (("child_off", "child_off"), ("child_tok", "child_tok"), ("child_node", "child_node"),
                         ("word_off", "word_off"), ("node_words", "words"), ("word_lm", "word_lm"), ("smear", "smear")):
                setattr(s, f, d[k].data_ptr())
            s.num_nodes, s.max_words = self.num_nodes, self.max_words
            d["struct"] = s
            self._dev[key] = d
        return self._dev[key]
