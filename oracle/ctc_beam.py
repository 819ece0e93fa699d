"""Oracle: frame-synchronous CTC prefix beam search with shallow LM fusion, in float64 numpy / Python.

TEST INFRASTRUCTURE ONLY.  The same statement as espresso_b200/csrc/ctc_beam.cu (and include/espresso_b200.h):

  hypothesis: prefix y, pb / pnb (log-prob of ending in blank / non-blank), lm (sum over its tokens of
              lm_weight * log P_LM(v | prefix) + word_score); score = logaddexp(pb, pnb) + lm.
  start:      one empty prefix, pb = 0, pnb = -inf.
  per frame t < in_len, lp = log_softmax(logits[t]):
    tokens    the K best tokens by logit (ties: lower id first), never blank or an excluded id;
    stay      pb' = lae(pb, pnb) + lp[blank]; pnb' = pnb + lp[last(y)] if y is non-empty;
    extend v  ext = (pb if v == last(y) else lae(pb, pnb)) + lp[v] -> y+v with pnb = ext, pb = -inf,
              lm += lm_weight * log P_LM(v | y) + word_score;
    merge     if y+v is a live hypothesis h', ext is log-added into pnb'(h') and the candidate disappears;
    prune     candidates below best - threshold are dropped; the best `beam` remain, ordered by (score desc,
              candidate index asc) with candidate index h * (K + 1) + j (j = 0 stay, j = 1..K extensions in rank
              order); the k-th becomes slot k of the next frame.
  end:        + lm_weight * log P_LM(eos | y) when an LM is fused; sort by (score desc, slot asc).

The LM is a callback lm_fn(prefix tuple) -> log-probabilities over the CTC vocabulary.  `dtype` selects the float type
of every arithmetic step (float64 for the oracle; oracle/ctc_beam_ops.py runs the same statement in float32)."""
import math
from collections import namedtuple

import numpy as np

Hyp = namedtuple("Hyp", "y pb pnb lm frames")
NEG = -math.inf


def topk_tokens(x, K, blank, exclude=()):
    """x [..., V] logits -> int64 [..., K]: the K best allowed tokens by (logit desc, id asc), -1 where fewer exist."""
    x = np.asarray(x, dtype=np.float64)
    V = x.shape[-1]
    bad = np.zeros(V, dtype=bool)
    for e in (blank,) + tuple(exclude):
        if e is not None and 0 <= e < V:
            bad[e] = True
    ids = np.broadcast_to(np.arange(V), x.shape)
    order = np.lexsort((ids, -x, np.broadcast_to(bad, x.shape)), axis=-1)[..., :K]
    tok = order.astype(np.int64)
    tok[bad[order]] = -1
    if K > V:
        tok = np.concatenate([tok, np.full(x.shape[:-1] + (K - V,), -1, dtype=np.int64)], axis=-1)
    return tok


def log_softmax(x, dtype=np.float64):
    x = np.asarray(x, dtype=dtype)
    m = x.max(axis=-1, keepdims=True)
    return (x - (m + np.log(np.exp(x - m).sum(axis=-1, keepdims=True)))).astype(dtype)


def _lae(a, b, dt):
    return dt(np.logaddexp(dt(a), dt(b)))


def initial(dt=np.float64):
    return [Hyp((), dt(0.0), dt(NEG), dt(0.0), ())]


def step(hyps, t, lp, lp_blank, tok, beam, threshold=math.inf, lm_fn=None, lm_weight=0.0, word_score=0.0, dt=np.float64):
    """One frame.  hyps: live hypotheses in slot order; lp: log-probs of the frame [V]; lp_blank: the blank's; tok: its K
    ranked tokens (-1 = none).  Returns (new hypotheses in slot order, [(source slot, appended token or -1)] per new slot)."""
    K = len(tok)
    index = {h.y: i for i, h in enumerate(hyps)}
    lp = np.asarray(lp, dtype=dt)
    spb = [dt(_lae(h.pb, h.pnb, dt) + dt(lp_blank)) for h in hyps]
    spnb = [dt(h.pnb + lp[h.y[-1]]) if h.y else dt(NEG) for h in hyps]
    merge = {}
    cands = []  # (score, candidate index, hypothesis, source slot, token)
    lw, ws = dt(lm_weight), dt(word_score)
    for i, h in enumerate(hyps):
        lml = None if lm_fn is None else np.asarray(lm_fn(h.y), dtype=dt)
        for j, v in enumerate(tok, 1):
            v = int(v)
            if v < 0:
                continue
            e = dt((h.pb if (h.y and v == h.y[-1]) else _lae(h.pb, h.pnb, dt)) + lp[v])
            y2 = h.y + (v,)
            if y2 in index:
                merge[index[y2]] = e
                continue
            lm = dt(h.lm + ws)
            if lml is not None:
                lm = dt(lm + dt(lw * lml[v]))
            cands.append((dt(e + lm), i * (K + 1) + j, Hyp(y2, dt(NEG), e, lm, h.frames + (t,)), i, v))
    for i, h in enumerate(hyps):
        pnb = _lae(spnb[i], merge.get(i, dt(NEG)), dt)
        cands.append((dt(_lae(spb[i], pnb, dt) + h.lm), i * (K + 1), Hyp(h.y, spb[i], pnb, h.lm, h.frames), i, -1))
    cands = [c for c in cands if c[0] > NEG and not np.isnan(c[0])]
    if not cands:
        return [], []
    best = max(c[0] for c in cands)
    floor_ = dt(best - dt(threshold))
    cands = sorted((c for c in cands if not c[0] < floor_), key=lambda c: (-c[0], c[1]))[:beam]
    return [c[2] for c in cands], [(c[3], c[4]) for c in cands]


def finish(hyps, lm_fn=None, lm_weight=0.0, eos=None, dt=np.float64):
    """-> [(tokens, score, frames)] sorted by (score desc, slot asc)."""
    out = []
    for k, h in enumerate(hyps):
        s = dt(_lae(h.pb, h.pnb, dt) + h.lm)
        if lm_fn is not None:
            s = dt(s + dt(dt(lm_weight) * dt(np.asarray(lm_fn(h.y), dtype=dt)[eos])))
        out.append((s, k, h))
    out.sort(key=lambda c: (-c[0], c[1]))
    return [(c[2].y, float(c[0]), c[2].frames) for c in out]


def search(logits, beam, K, blank, exclude=(), threshold=math.inf, lm_fn=None, lm_weight=0.0, word_score=0.0, eos=None):
    """logits [T, V] (the sentence's frames) -> every final hypothesis as (tokens, score, frames), best first."""
    x = np.asarray(logits, dtype=np.float64)
    lps = log_softmax(x)
    toks = topk_tokens(x, K, blank, exclude)
    hyps = initial()
    for t in range(x.shape[0]):
        hyps, _ = step(hyps, t, lps[t], lps[t, blank], toks[t], beam, threshold, lm_fn, lm_weight, word_score)
    return finish(hyps, lm_fn, lm_weight, eos)
