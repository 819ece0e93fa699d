"""Oracle: plain-PyTorch (CPU, fp32) statement of the transducer beam-search kernels (espresso_b200/csrc/
transducer_beam.cu), with the signatures of their wrappers in espresso_b200/ops.py (rnnt_beam_*).

TEST INFRASTRUCTURE ONLY.  GPU tests compare each kernel with the function of the same name here; CPU tests
monkeypatch these in for `espresso_b200.ops` to run BatchedAdaptiveExpansionSearch without a GPU.  The search state
`st` is the dict of flat tables espresso_b200.tools.transducer_beam_search_decoder.beam_state allocates; these
statements read and update it in place exactly as the kernels do.  Ties rank by (value desc, candidate index asc)
everywhere.  Prefix hashes are esp_hash_u64 of csrc/common.cuh (oracle/dropout_rng.hash_u64).
"""
import numpy as np
import torch

from oracle import dropout_rng as _rng


def _rank(keys):
    """Positions of `keys` (a list of floats) ordered by (key desc, index asc); NaN ranks last."""
    return sorted(range(len(keys)), key=lambda i: (-keys[i] if keys[i] == keys[i] else float("inf"), i))


def rnnt_beam_lprobs(logits, V, scores, k, blank, temperature=1.0, eos=-1, fold_eos=False, lm_logits=None, lm_weight=0.0,
                     no_blank_in_lm=False):
    """transducer_beam_search_decoder.py:465-601 (one expansion's log-probs): log_softmax(logits / temperature), the LM's
    non-blank fusion renormalised to the transducer's non-blank mass, eos folded into blank, + the row's score; the row's
    top k as (values fp32 [n, k], tokens int32 [n, k]) and its unfused, unfolded blank log-prob fp32 [n]."""
    lp = torch.log_softmax(logits[:, :V].float() / temperature, dim=-1)
    lpb = lp[:, blank].clone()
    if lm_logits is not None:
        nb = torch.ones(V, dtype=torch.bool)
        nb[blank] = False
        nb = nb.to(lp.device)
        lm_lp = torch.log_softmax(lm_logits[:, :V - int(no_blank_in_lm)].float(), dim=-1)
        if not no_blank_in_lm:
            lm_lp = lm_lp[:, nb]
        lp_nb = lp[:, nb]
        fused = lp_nb + lm_weight * lm_lp
        lp[:, nb] = fused + (lp_nb.exp().sum(1).log() - fused.exp().sum(1).log())[:, None]
    if fold_eos:
        lp[:, blank] = torch.logaddexp(lp[:, blank], lp[:, eos])
        lp[:, eos] = float("-inf")
    tot = lp + scores.float()[:, None]
    val, tok = torch.sort(tot, dim=1, descending=True, stable=True)
    return val[:, :k].contiguous(), tok[:, :k].to(torch.int32).contiguous(), lpb


def _node_hash(st, b, parent, tok):
    P = st["P"]
    return int(_rng.hash_u64(int(st["p_hash"][b * P + parent]) & ((1 << 64) - 1), [tok])[0].astype(np.int64))


def _push_node(st, b, parent, tok):
    P = st["P"]
    n = int(st["npool"][b])
    assert n < P, "transducer beam search: prefix node pool full"
    st["p_parent"][b * P + n] = parent
    st["p_tok"][b * P + n] = tok
    st["p_len"][b * P + n] = int(st["p_len"][b * P + parent]) + 1
    st["p_hash"][b * P + n] = _node_hash(st, b, parent, tok)
    st["npool"][b] = n + 1
    return n


def _ancestor(st, b, node, up):
    for _ in range(up):
        node = int(st["p_parent"][st["P"] * b + node])
    return node


def rnnt_beam_prefix_merge(st, t, alpha):
    """transducer_beam_search_decoder.py:270-463 (prefix search, first half): per utterance still inside its frames, order
    the rows by length (longest first), reset the frame's counters, and list every pair (j, i) -- i a prefix of j, at most
    alpha tokens shorter, j outer and i inner in that order -- with the ring rows (age * ring_stride + state row) and
    tokens of its path steps."""
    B, K, S, Pm = st["B"], st["K"], st["S"], st["Pm"]
    for b in range(B):
        n = int(st["nrow"][b])
        active = t < int(st["nframes"][b])
        st["nlive"][b] = n if active else 0
        st["na"][b] = 0
        st["m_npair"][b] = 0
        rows = range(b * K, b * K + K)
        if not active:
            for s in rows:
                st["srow"][s] = s
                st["fsrc"][s] = s
            continue
        lens = [int(st["len"][b * K + s]) for s in range(n)]
        order = _rank([float(x) for x in lens])
        for key in ("score", "nemit", "len", "node"):
            v = st[key][b * K: b * K + n].clone()
            st[key][b * K: b * K + n] = v[order]
        for p in range(K):
            st["srow"][b * K + p] = b * K + (order[p] if p < n else p)
        npair = nstep = 0
        for pj in range(n - 1):
            for pi in range(pj + 1, n):
                li, lj = int(st["len"][b * K + pi]), int(st["len"][b * K + pj])
                if not (li < lj <= li + alpha):
                    continue
                nj, ni = int(st["node"][b * K + pj]), int(st["node"][b * K + pi])
                if int(st["p_hash"][b * st["P"] + _ancestor(st, b, nj, lj - li)]) != int(st["p_hash"][b * st["P"] + ni]):
                    continue
                base = b * Pm * 4 + npair * 4
                st["m_pair"][base: base + 4] = torch.tensor([pj, pi, b * S + nstep, lj - li], dtype=torch.int32)
                # step at position pos emits j's token at depth pos + 2 from the decoder output at pos: i's newest (age 0)
                # for pos = li - 1, then j's at age lj - 1 - pos
                for pos in range(li - 1, lj - 1):
                    src, age = (pi, 0) if pos == li - 1 else (pj, lj - 1 - pos)
                    st["m_ring"][b * S + nstep] = age * st["ring_stride"] + int(st["srow"][b * K + src])
                    st["m_tok"][b * S + nstep] = int(st["p_tok"][b * st["P"] + _ancestor(st, b, nj, lj - pos - 2)])
                    nstep += 1
                npair += 1
        st["m_npair"][b] = npair


def rnnt_beam_merge_scores(logits, V, st, temperature=1.0, blank=0, lm_logits=None, lm_weight=0.0, no_blank_in_lm=False):
    """transducer_beam_search_decoder.py:270-463 (prefix search, second half): each listed pair's path score -- i's score
    plus, per step, the step's log-prob of j's token (with an LM: + lm_weight * its LM log-prob + the fusion's
    renormalisation term) -- is log-added into j, pairs in the listed order."""
    B, K, Pm = st["B"], st["K"], st["Pm"]
    lp = torch.log_softmax(logits[:, :V].float() / temperature, dim=-1)
    if lm_logits is not None:
        nb = torch.ones(V, dtype=torch.bool)
        nb[blank] = False
        nb = nb.to(lp.device)
        lm_lp = torch.log_softmax(lm_logits[:, :V - int(no_blank_in_lm)].float(), dim=-1)
        lp_nb = lp[:, nb]
        fused = lp_nb + lm_weight * (lm_lp if no_blank_in_lm else lm_lp[:, nb])
        scale = lp_nb.exp().sum(1).log() - fused.exp().sum(1).log()
    for b in range(B):
        for q in range(int(st["m_npair"][b])):
            pj, pi, s0, ns = st["m_pair"][b * Pm * 4 + q * 4: b * Pm * 4 + q * 4 + 4].tolist()
            sc = st["score"][b * K + pi].clone()
            for s in range(s0, s0 + ns):
                tok = int(st["m_tok"][s])
                sc = sc + lp[s, tok]
                if lm_logits is not None:
                    lt = tok - 1 if (no_blank_in_lm and tok > blank) else tok
                    sc = sc + lm_weight * lm_lp[s, lt] + scale[s]
            st["score"][b * K + pj] = torch.logaddexp(st["score"][b * K + pj], sc)


def _combine(st, b, rnd, beam, normalize, blank, lpb, final):
    K, A, BK = st["K"], st["A"], st["B"] * st["K"]
    cand = [(float(st["a_score"][b * A + q]), int(st["a_nemit"][b * A + q]), int(st["a_len"][b * A + q]),
             int(st["a_node"][b * A + q]), int(st["a_src"][b * A + q])) for q in range(int(st["na"][b]))]
    if final:
        for s in range(b * K, b * K + int(st["nlive"][b])):
            cand.append((float(np.float32(float(st["score"][s]) + float(lpb[s]))), int(st["nemit"][s]) + 1, int(st["len"][s]),
                         int(st["node"][s]), (rnd + 1) * BK + s))
    with np.errstate(divide="ignore", invalid="ignore"):
        keys = [float(np.float32(c[0]) / np.float32(c[1])) if normalize else c[0] for c in cand]
    keep = _rank(keys)[:beam]
    for p, c in enumerate(keep):
        s = b * K + p
        st["score"][s], st["nemit"][s], st["len"][s], st["node"][s], st["fsrc"][s] = cand[c]
    st["nrow"][b] = len(keep)
    st["nlive"][b] = 0


def rnnt_beam_select(val, tok, lpb, st, rnd, beam, blank, gamma=None, normalize=True, final=False):
    """transducer_utils.py select_k_expansions and transducer_beam_search_decoder.py:465-601 (one expansion round) per
    utterance with live rows.  Not final: the rows' proposals (candidate index row * k + rank) lose those more than gamma
    below their row's best, the best k remain (ranked by score / nemit when normalising); blank ones are set aside with
    their row's state reference, non-blank ones become the next round's rows (a prefix node each, parent = the state row
    to advance).  An utterance left without a non-blank proposal ends its frame: the best `beam` set-aside entries
    become its rows.  Final (after the last round's predictor step): the live rows pay their blank log-prob and compete
    with the set-aside entries for the `beam` rows.  Writes fsrc, the state reference of each new row."""
    B, K, A, BK = st["B"], st["K"], st["A"], st["B"] * st["K"]
    k = val.size(1)
    for b in range(B):
        n = int(st["nlive"][b])
        if n == 0:
            continue
        if final:
            _combine(st, b, rnd, beam, normalize, blank, lpb, True)
            continue
        rows = list(range(b * K, b * K + n))
        toks = [[int(tok[s, q]) for q in range(k)] for s in rows]
        all_blank = all(x == blank for r in toks for x in r)
        cand, keys = [], []
        for r, s in enumerate(rows):
            best = float(val[s, 0])
            for q in range(k):
                v = float(val[s, q])
                if gamma is not None and not v >= best - gamma:
                    continue
                ne = int(st["nemit"][s]) + (0 if all_blank else 1)
                cand.append((r, q, v, ne))
                with np.errstate(divide="ignore", invalid="ignore"):
                    keys.append(float(np.float32(v) / np.float32(ne)) if normalize else v)
        keep = [cand[i] for i in _rank(keys)[:k]]
        old = {key: st[key][b * K: b * K + n].clone() for key in ("nemit", "len", "node", "srow")}
        m = 0
        for (r, q, v, ne) in keep:
            x = toks[r][q]
            if x == blank:
                a = b * A + int(st["na"][b])
                st["a_score"][a], st["a_nemit"][a], st["a_len"][a] = v, ne, int(old["len"][r])
                st["a_node"][a], st["a_src"][a] = int(old["node"][r]), rnd * BK + int(old["srow"][r])
                st["na"][b] += 1
            else:
                s = b * K + m
                st["score"][s], st["nemit"][s], st["len"][s] = v, ne, int(old["len"][r]) + 1
                st["node"][s] = _push_node(st, b, int(old["node"][r]), x)
                st["parent"][s], st["prev"][s], st["srow"][s] = int(old["srow"][r]), x, s
                m += 1
        st["nlive"][b] = m
        if m == 0:
            _combine(st, b, rnd, beam, normalize, blank, lpb, False)


def rnnt_beam_finalize(st, pad):
    """transducer_beam_search_decoder.py:465-601 (end of search): scores / (len - 1), sorted best first; each row's tokens
    (bos dropped) backtracked from the prefix node pool.  Returns (tokens int64 [B, K, L] pad-filled, scores fp32 [B, K],
    lens int32 [B, K] (tokens per row, 0 for missing rows)) with L = the longest row."""
    B, K, P = st["B"], st["K"], st["P"]
    L = max([int(st["len"][b * K + s]) - 1 for b in range(B) for s in range(int(st["nrow"][b]))] + [1])
    out = torch.full((B, K, L), pad, dtype=torch.int64)
    sc = torch.full((B, K), float("-inf"))
    lens = torch.zeros(B, K, dtype=torch.int32)
    for b in range(B):
        n = int(st["nrow"][b])
        with np.errstate(divide="ignore", invalid="ignore"):
            norm = [float(np.float32(float(st["score"][b * K + s])) / np.float32(int(st["len"][b * K + s]) - 1)) for s in range(n)]
        for p, s in enumerate(_rank(norm)):
            ln = int(st["len"][b * K + s]) - 1
            sc[b, p], lens[b, p] = norm[s], ln
            node = int(st["node"][b * K + s])
            for d in range(ln - 1, -1, -1):
                out[b, p, d] = int(st["p_tok"][b * P + node])
                node = int(st["p_parent"][b * P + node])
    return out, sc, lens
