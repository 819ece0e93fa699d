"""Lexical prefix tree over the word dictionary, flattened for the look-ahead LM fusion kernels.

Same information as the reference's tree (espresso/tools/lexical_prefix_tree.py:13-67: children by subword id, the word
ending at a node, and the contiguous range (first - 1, last) of word ids below it -- word dictionaries are in lexical
order) and its tensorised form (espresso/tools/tensorized_prefix_tree.py:15-108: node 0 = "outside the lexicon",
node 1 = root).  The reference stores children as a dense int64 [nodes, max_out_degree] table, which for a 5 000-unit
subword vocabulary and ~10^5 nodes is gigabytes; here the edges are CSR (offsets + (subword, child) pairs sorted by
subword), 12 bytes per node, and csrc/lookahead.cu walks them directly."""
import numpy as np
import torch

from ..data.encoders import tokenize


def csr_edges(edge, n):
    """{(parent node, subword id): child node} over n nodes -> int32 (child_off [n + 1], child_tok, child_node), the
    edges of each node sorted by subword id."""
    keys = sorted(edge)             # by parent, then subword id
    off = np.zeros(n + 1, dtype=np.int64)
    for parent, _ in keys:
        off[parent + 1] += 1
    i32 = lambda a: np.asarray(a, dtype=np.int32)  # noqa: E731
    return i32(np.cumsum(off)), i32([k[1] for k in keys]), i32([edge[k] for k in keys])


class TensorizedPrefixTree:
    none_id, root_id = 0, 1

    def __init__(self, child_off, child_tok, child_node, node_word, node_lo, node_hi):
        self.child_off, self.child_tok, self.child_node = child_off, child_tok, child_node
        self.node_word, self.node_lo, self.node_hi = node_word, node_lo, node_hi
        self._dev = {}

    @property
    def num_nodes(self):
        return len(self.node_word)

    def max_out_degree(self):
        return int(np.diff(self.child_off).max()) if self.num_nodes else 0

    @classmethod
    def build(cls, word_dict, subword_dict, subword_tokenizer=None):
        """Words containing a subword the subword dictionary does not know, and <pad> / </s> / <unk>, stay out of the tree
        (lexical_prefix_tree.py:43-58)."""
        specials = {word_dict.pad(), word_dict.eos(), word_dict.unk()}
        if 0 not in specials:
            raise ValueError("word id 0 must be a special symbol (the ranges store first_word_id - 1)")
        if subword_tokenizer is None:
            non_lang = getattr(subword_dict, "non_lang_syms", None)
            subword_tokenizer = lambda w: tokenize(w, non_lang_syms=non_lang).split(" ")  # noqa: E731
        unk = subword_dict.unk()
        edge = {}                       # (parent node, subword id) -> node
        word, lo, hi = [-1, -1], [word_dict.pad(), 0], [word_dict.pad(), len(word_dict) - 1]
        for widx in range(len(word_dict)):
            if widx in specials:
                continue
            ids = [subword_dict.index(s) for s in subword_tokenizer(word_dict[widx])]
            if not ids or any(i == unk for i in ids):
                continue
            node = cls.root_id
            for i in ids:
                nxt = edge.get((node, i))
                if nxt is None:
                    nxt = edge[(node, i)] = len(word)
                    word.append(-1)
                    lo.append(widx - 1)
                    hi.append(widx)
                else:
                    lo[nxt] = min(lo[nxt], widx - 1)
                    hi[nxt] = max(hi[nxt], widx)
                node = nxt
            word[node] = widx
        i32 = lambda a: np.asarray(a, dtype=np.int32)  # noqa: E731
        return cls(*csr_edges(edge, len(word)), i32(word), i32(lo), i32(hi))

    def step(self, node, subword):
        """Host transition (tests / debugging): child of `node` labelled `subword`, else none_id."""
        e0, e1 = self.child_off[node], self.child_off[node + 1]
        j = e0 + int(np.searchsorted(self.child_tok[e0:e1], subword))
        return int(self.child_node[j]) if j < e1 and self.child_tok[j] == subword else self.none_id

    def to(self, device):
        """Device copies (int32), cached per device."""
        key = str(device)
        if key not in self._dev:
            names = ("child_off", "child_tok", "child_node", "node_word", "node_lo", "node_hi")
            self._dev[key] = {k: torch.from_numpy(np.ascontiguousarray(getattr(self, k))).to(device) for k in names}
            for k in ("child_tok", "child_node"):       # an edge-less lexicon still needs valid pointers
                if self._dev[key][k].numel() == 0:
                    self._dev[key][k] = torch.zeros(1, dtype=torch.int32, device=device)
        return self._dev[key]
