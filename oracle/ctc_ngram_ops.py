"""Oracle: plain numpy statement of the n-gram ops in espresso_b200/ops.py (ngram_score, ctc_ngram_workspace,
ctc_ngram_search, ctc_ngram_finalize), same signatures, fp32 arithmetic.

TEST INFRASTRUCTURE ONLY.  CPU tests monkeypatch these in for `espresso_b200.ops` (next to oracle/ops_ref.py and
oracle/ctc_beam_ops.py) to run the host orchestration of espresso_b200/tools/ctc_decoder.py without a GPU.  `probe` is
the fp32 restatement of the kernels' n-gram walk over the tables the host builder made (NgramLanguageModel's arrays);
the searches are oracle/ctc_beam.py's step (lexicon-free) and oracle/ngram.py's lexicon_step run in float32."""
import numpy as np
import torch

F32 = np.float32


def probe(lm, s, w):
    """(log10 P(w | state s), next state) in fp32, walking s and its suffix links as esp_ngram_score does."""
    acc = F32(0.0)
    while s >= 0:
        lo, hi = int(lm.child_lo[s]), int(lm.child_hi[s])
        j = lo + int(np.searchsorted(lm.word[lo:hi], w))
        if j < hi and lm.word[j] == w:
            order = int(np.searchsorted(lm.order_off, j, side="right"))
            return F32(acc + lm.prob[j]), (j if order < lm.order else int(lm.suffix[j]))
        acc = F32(acc + lm.backoff[s])
        s = int(lm.suffix[s])
    return F32(acc + lm.prob[w]), (w if lm.order > 1 else -1)


def state_of(lm, words):
    s = lm.start
    for w in words:
        _, s = probe(lm, s, w)
    return s


def ngram_score(lm, states, words):
    out = [probe(lm, int(s), int(w)) for s, w in zip(states.tolist(), words.tolist())]
    return (torch.tensor([o[0] for o in out], dtype=torch.float32), torch.tensor([o[1] for o in out], dtype=torch.int32))


def ctc_ngram_workspace(B, T, beam, device):
    return {"B": B, "T": T, "beam": beam, "hyps": None}


def _word_fn(lm, word_lm):
    """lexicon word ids -> fp32 log10 P from the tables; word id -1 stands for </s>."""
    cache = {}

    def fn(hist, w):
        if (hist, w) not in cache:
            cache[(hist, w)] = probe(lm, state_of(lm, [int(word_lm[x]) for x in hist]), lm.eos if w < 0 else int(word_lm[w]))[0]
        return cache[(hist, w)]

    return fn


def _token_fn(lm, tok_word):
    """lexicon-free: prefix -> fp32 log10 P(. | prefix) over the CTC vocabulary."""
    tw = [int(x) for x in tok_word.tolist()]
    cache = {}

    def fn(y):
        if y not in cache:
            s = state_of(lm, [tw[v] for v in y])
            cache[y] = np.array([probe(lm, s, w)[0] for w in tw], dtype=F32)
        return cache[y]

    return fn


def _lexicon(trie, lm):
    from oracle import ngram as N

    if trie.smear is None:
        trie.smear = trie.compute_smear(np.array([probe(lm, lm.start, int(w))[0] for w in trie.word_lm], dtype=F32))
    lex = N.Lexicon.__new__(N.Lexicon)
    lex.words = list(range(len(trie.words)))
    paths = {0: ()}
    for n in range(trie.num_nodes):  # parents come before children
        for e in range(trie.child_off[n], trie.child_off[n + 1]):
            paths[int(trie.child_node[e])] = paths[n] + (int(trie.child_tok[e]),)
    lex.ends = {paths[n]: [int(w) for w in trie.node_words[trie.word_off[n]:trie.word_off[n + 1]]]
                for n in range(trie.num_nodes) if trie.word_off[n + 1] > trie.word_off[n]}
    lex.prefixes = set(paths.values()) - {()}
    lex.inner = {paths[n] for n in range(1, trie.num_nodes) if trie.child_off[n + 1] > trie.child_off[n]}
    lex.max_words = trie.max_words
    lex.smear = {paths[n]: F32(trie.smear[n]) for n in range(trie.num_nodes)}
    return lex


def ctc_ngram_search(logits, V, in_lens, frames, beam, beam_threshold, workspace, lm, tok_word=None, lexicon=None,
                     lm_weight=0.0, word_score=0.0):
    from oracle import ctc_beam as O
    from oracle import ngram as N

    B, T, _ = logits.shape
    lse, lpb, tok, _ = frames
    x = logits[..., :V].float().numpy()
    lex = _lexicon(lexicon, lm) if lexicon is not None else None
    fn = _word_fn(lm, lexicon.word_lm) if lexicon is not None else _token_fn(lm, tok_word)
    workspace["fn"], workspace["tw"] = fn, tok_word
    workspace["hyps"] = []
    for b in range(B):
        hyps = N.lexicon_initial(F32) if lex is not None else O.initial(F32)
        for t in range(min(T, int(in_lens[b]))):
            lp = (x[b, t] - lse[b, t].numpy()).astype(F32)
            if lex is not None:
                hyps, _ = N.lexicon_step(hyps, t, lp, lpb[b, t].numpy(), tok[b, t].numpy(), beam, F32(beam_threshold), lex, fn,
                                         lm_weight, word_score, F32)
            else:
                hyps, _ = O.step(hyps, t, lp, lpb[b, t].numpy(), tok[b, t].numpy(), beam, F32(beam_threshold), fn, lm_weight,
                                 word_score, F32)
        workspace["hyps"].append(hyps)


def _finish_free(hyps, tok_word, lm, lm_weight):
    """oracle/ctc_beam.py's finish with the n-gram: + lm_weight * log10 P(</s> | y), by (score desc, slot asc)."""
    tw = [int(x) for x in tok_word.tolist()]
    out = []
    for k, h in enumerate(hyps):
        s = F32(np.logaddexp(F32(h.pb), F32(h.pnb)) + h.lm)
        s = F32(s + F32(F32(lm_weight) * probe(lm, state_of(lm, [tw[v] for v in h.y]), lm.eos)[0]))
        out.append((s, k, h))
    out.sort(key=lambda c: (-c[0], c[1]))
    return [(c[2].y, float(c[0]), c[2].frames) for c in out]


def ctc_ngram_finalize(in_lens, T, V, beam, nbest, workspace, lm, lexicon=None, lm_weight=0.0, pad=1, want_frames=False):
    from oracle import ctc_beam as O
    from oracle import ngram as N

    B = in_lens.numel()
    tokens = torch.full((B, nbest, T), pad, dtype=torch.int32)
    frames = torch.full((B, nbest, T), -1, dtype=torch.int32)
    lens = torch.zeros(B, nbest, dtype=torch.int32)
    scores = torch.full((B, nbest), float("-inf"))
    for b in range(B):
        hyps = workspace["hyps"][b]
        if lexicon is not None:
            res = [r[:3] for r in N.lexicon_finish(hyps, workspace["fn"], lm_weight, -1, F32)]
        else:
            res = _finish_free(hyps, workspace["tw"], lm, lm_weight)
        for r, (y, s, fr) in enumerate(res[:nbest]):
            tokens[b, r, :len(y)] = torch.tensor(y, dtype=torch.int32)
            frames[b, r, :len(y)] = torch.tensor(fr, dtype=torch.int32)
            lens[b, r] = len(y)
            scores[b, r] = s
    return tokens, lens, scores, (frames if want_frames else None)
