"""Oracle: the search options of the reference's SequenceGenerator, restated on the CPU.  TEST INFRASTRUCTURE ONLY.

Two layers:
  * per-op statements of the native entry points (esp_beam_block_ngrams, esp_beam_prefix, esp_beam_diverse_groups,
    esp_beam_sibling_topk) with the signatures of their espresso_b200.ops wrappers, used by the GPU kernel tests and, through
    monkeypatching, to run the product generator's host orchestration on the CPU;
  * `generate`: oracle/beam.generate's restatement of fairseq/sequence_generator.py extended by prefix tokens (:414-424,
    _prefix_tokens :623-657, batch compaction of the prefix :536), n-gram blocking (:448-449) and the search classes
    DiverseBeamSearch / DiverseSiblingsSearch (fairseq/search.py:551-618, 745-810).  oracle/pin_search_strategies.py pins it
    against the real reference -> tests/golden/search_strategies.npz.

Where torch.topk leaves ties unordered, every top-k here takes (value descending, index ascending), as the kernels do.
N-gram blocking compares the window that ends at the current step (the reference's CUDA extension,
fairseq/clib/cuda/ngram_repeat_block_cuda_kernel.cu, and its Python path when handed tokens[:, :step + 1]).
"""
import math

import numpy as np
import torch

from oracle.beam import topk_lex
from oracle.dropout_rng import hash_u64

NEG = -math.inf


# ---------------------------------------------------------------------------------------------------------------------
# per-op statements
# ---------------------------------------------------------------------------------------------------------------------
def beam_block_ngrams(tokens, step, n, lprobs, V):
    tail = step - n + 2
    for r, row in enumerate(tokens[:, : step + 1].tolist()):
        for i in range(max(tail, 0)):
            if row[i: i + n - 1] == row[tail: tail + n - 1] and 0 <= row[i + n - 1] < V:
                lprobs[r, row[i + n - 1]] = NEG
    return lprobs


def beam_prefix(prefix, step, beam, pad, eos, cand, V, st):
    for s in range(prefix.shape[0]):
        pt = int(prefix[s, step])
        if pt == pad:
            continue
        rows = slice(s * beam, (s + 1) * beam)
        keep = cand[rows, pt].clone()
        cand[rows] = NEG
        cand[rows, pt] = keep
        if pt == eos:  # replicate_first_beam (:649-652)
            cand[rows] = cand[s * beam].clone()
            st.tokens[rows] = st.tokens[s * beam].clone()
            st.scores[rows] = st.scores[s * beam].clone()
    return cand


def beam_diverse_groups(lprobs, prev_scores, bsz, beam, V, groups, Kg, strength):
    """DiverseBeamSearch.step over the merged log-probs (no cumulative scores in `lprobs`)."""
    lp = lprobs.float().view(bsz, beam, V)
    div = torch.zeros(bsz, V)
    S, T, B = [], [], []
    for g in range(groups):
        x = lp[:, g::groups, :]
        if g > 0:
            x = x + div.unsqueeze(1) * (-strength)
        if prev_scores is None:
            x = x[:, :1, :]
        else:
            x = x + prev_scores.float().view(bsz, beam)[:, g::groups].unsqueeze(-1)
        s, flat = topk_lex(x.reshape(bsz, -1), Kg)
        S.append(s)
        T.append(flat % V)
        B.append((flat // V) * groups + g)
        div.scatter_add_(1, flat % V, torch.ones(bsz, Kg))
    s = torch.stack(S, dim=2).view(bsz, -1)
    return s, torch.stack(T, dim=2).view(bsz, -1).int(), torch.stack(B, dim=2).view(bsz, -1).int()


def beam_sibling_topk(cand, bsz, beam, V, k, rate):
    """DiverseSiblingsSearch.step at step > 0 over candidates that already hold the cumulative scores."""
    s1, i1 = topk_lex(cand.float().view(bsz * beam, V), k)
    s1 = s1 - torch.arange(1, k + 1, dtype=torch.float32) * rate
    s, flat = topk_lex(s1.view(bsz, beam * k), k)
    b = flat // k
    t = torch.gather(i1.view(bsz, beam * k), 1, flat)
    return s, t.int(), b.int()


_FIX = np.float32(2.0 ** 40)


def sample_uniform_hash(seed, step, row, draw):
    """The 64-bit hash behind one draw of esp_beam_sample."""
    return int(hash_u64(int(hash_u64(seed, step)), (int(row) << 16) | int(draw)))


def beam_sample(lprobs, prev_scores, bsz, beam, V, topk, topp, seed, step, sent_ids=None):
    """Sampling.step (fairseq/search.py:621-742) as esp_beam_sample draws it: the kept set by exact fixed-point masses in
    (p descending, token ascending) order, then an inverse-CDF draw in token order from the counter RNG.  sent_ids: the
    sentence of each local sentence in the batch whose row numbers key the draws (default: the same)."""
    seed = int(seed.reshape(-1)[0]) if torch.is_tensor(seed) else int(seed)
    lp = lprobs.float().view(bsz * beam, V)
    S, T, B = torch.empty(bsz, beam), torch.empty(bsz, beam, dtype=torch.int32), torch.empty(bsz, beam, dtype=torch.int32)
    for o in range(bsz * beam):
        s, j = divmod(o, beam)
        row = o if prev_scores is not None else s * beam
        p = torch.exp(lp[row]).numpy()
        W = [int(np.float32(x) * _FIX) for x in p]
        order = sorted(range(V), key=lambda v: (-float(p[v]), v))
        if topp > 0:
            limit, mass = int(np.float32(topp) * _FIX), W
        elif 0 < topk < V:
            limit, mass = int(topk), [1] * V
        else:
            limit, mass = None, None
        keep = [True] * V
        if limit is not None:
            before = 0
            for v in order:
                keep[v] = before < limit
                before += mass[v]
        wtot = sum(W[v] for v in range(V) if keep[v])
        g = row if sent_ids is None else int(sent_ids[row // beam]) * beam + row % beam
        h = sample_uniform_hash(seed, step, g, 0 if prev_scores is not None else j)
        t_, pick, cum = (h * wtot) >> 64, -1, 0
        for v in range(V):
            if keep[v]:
                cum += W[v]
                if wtot > 0 and t_ < cum:
                    pick = v
                    break
        k = max(pick, 0)
        sc = torch.log(torch.tensor(p[k], dtype=torch.float32)) if pick >= 0 else torch.tensor(NEG)
        if prev_scores is not None:
            sc = sc + prev_scores.float()[o]
        S[s, j], T[s, j], B[s, j] = sc, k, j if prev_scores is not None else 0
    return S, T, B


# ---------------------------------------------------------------------------------------------------------------------
# the generator
# ---------------------------------------------------------------------------------------------------------------------
def generate(lprobs_fn, bsz, src_len, V, pad, unk, eos, beam_size=1, max_len_a=0, max_len_b=200, model_max_len=100, min_len=1,
             normalize_scores=True, len_penalty=1.0, unk_penalty=0.0, eos_factor=None, no_repeat_ngram_size=0, prefix_tokens=None,
             diverse_beam_groups=-1, diverse_beam_strength=0.5, diversity_rate=-1.0, sampling=False, sampling_topk=-1,
             sampling_topp=-1.0, sampling_seed=1):
    beam = min(beam_size, V - 1)
    max_len = min(int(max_len_a * src_len + max_len_b), model_max_len - 1)
    scores = torch.zeros(bsz * beam, max_len + 1)
    tokens = torch.full((bsz * beam, max_len + 2), pad, dtype=torch.long)
    tokens[:, 0] = eos
    cands_to_ignore = torch.zeros(bsz, beam, dtype=torch.bool)
    finalized = [[] for _ in range(bsz)]
    finished = [False] * bsz
    num_remaining = bsz
    cand_size = 2 * beam
    bbsz_offsets = (torch.arange(bsz) * beam).unsqueeze(1)
    cand_offsets = torch.arange(cand_size)
    reorder_state, batch_idxs = None, None
    orig = torch.arange(bsz)  # each remaining sentence's index in the original batch
    for step in range(max_len + 1):
        if reorder_state is not None and batch_idxs is not None:
            corr = batch_idxs - torch.arange(batch_idxs.numel())
            reorder_state.view(-1, beam).add_(corr.unsqueeze(-1) * beam)
        lprobs = lprobs_fn(step, tokens[:, : step + 1], reorder_state).clone().float()
        lprobs[lprobs != lprobs] = NEG
        lprobs[:, pad] = NEG
        lprobs[:, unk] -= unk_penalty
        if step >= max_len:
            lprobs[:, :eos] = NEG
            lprobs[:, eos + 1:] = NEG
        elif eos_factor is not None:
            dis = lprobs[:, eos] < eos_factor * lprobs.max(dim=1)[0]
            lprobs[dis, eos] = NEG
        if prefix_tokens is not None and step < prefix_tokens.size(1) and step < max_len:
            # _prefix_tokens (:623-657)
            prefix_toks = prefix_tokens[:, step].unsqueeze(-1).repeat(1, beam).view(-1)
            prefix_lprobs = lprobs.gather(-1, prefix_toks.unsqueeze(-1))
            prefix_mask = prefix_toks.ne(pad)
            lprobs[prefix_mask] = NEG
            lprobs[prefix_mask] = lprobs[prefix_mask].scatter(-1, prefix_toks[prefix_mask].unsqueeze(-1),
                                                              prefix_lprobs[prefix_mask])
            eos_mask = prefix_toks.eq(eos)
            if eos_mask.any():
                m = eos_mask.view(-1, beam)[:, 0]
                for t_ in (tokens, scores, lprobs):
                    v_ = t_.view(-1, beam, t_.size(-1))
                    v_[m] = v_[m][:, :1, :]
        elif step < min_len:
            lprobs[:, eos] = NEG
        if no_repeat_ngram_size > 0:
            beam_block_ngrams(tokens, step, no_repeat_ngram_size, lprobs, V)
        # the search step
        if sampling:  # one draw per hypothesis; the draws are keyed by the rows of the uncompacted batch
            cand_scores, cand_indices, cand_beams = beam_sample(lprobs, None if step == 0 else scores[:, step - 1], bsz, beam, V,
                                                                sampling_topk, sampling_topp, sampling_seed, step, sent_ids=orig)
            cand_indices, cand_beams = cand_indices.long(), cand_beams.long()
        elif diverse_beam_groups > 0:
            G = diverse_beam_groups
            Kg = min(2 * (beam // G), (V if step == 0 else beam // G * V) - 1)
            cand_scores, cand_indices, cand_beams = beam_diverse_groups(
                lprobs, None if step == 0 else scores[:, step - 1], bsz, beam, V, G, Kg, diverse_beam_strength)
            cand_indices, cand_beams = cand_indices.long(), cand_beams.long()
        elif diversity_rate > -1 and step > 0:
            lp = lprobs + scores[:, step - 1].unsqueeze(-1)
            cand_scores, cand_indices, cand_beams = beam_sibling_topk(lp, bsz, beam, V, min(2 * beam, beam * V - 1),
                                                                      diversity_rate)
            cand_indices, cand_beams = cand_indices.long(), cand_beams.long()
        else:
            lp = lprobs.view(bsz, -1, V)
            if step == 0:
                lp = lp[:, ::beam, :].contiguous()
            else:
                lp = lp + scores.view(bsz, beam, -1)[:, :, step - 1].unsqueeze(-1)
            cand_scores, flat = topk_lex(lp.view(bsz, -1), min(beam * 2, lp.view(bsz, -1).size(1) - 1))
            cand_beams, cand_indices = flat // V, flat % V
        cand_bbsz_idx = cand_beams + bbsz_offsets
        eos_mask = cand_indices.eq(eos) & cand_scores.ne(NEG)
        eos_mask[:, :beam][cands_to_ignore] = False
        eos_bbsz_idx = torch.masked_select(cand_bbsz_idx[:, :beam], eos_mask[:, :beam])
        finalized_sents = []
        if eos_bbsz_idx.numel() > 0:
            eos_scores = torch.masked_select(cand_scores[:, :beam], eos_mask[:, :beam])
            tok_clone = tokens.index_select(0, eos_bbsz_idx)[:, 1: step + 2].clone()
            tok_clone[:, step] = eos
            pos = scores.index_select(0, eos_bbsz_idx)[:, : step + 1].clone()
            pos[:, step] = eos_scores
            pos[:, 1:] = pos[:, 1:] - pos[:, :-1]
            if normalize_scores:
                eos_scores = eos_scores / (step + 1) ** len_penalty
            cum_unfin, prev = [], 0
            for f in finished:
                if f:
                    prev += 1
                else:
                    cum_unfin.append(prev)
            unfin_idx = eos_bbsz_idx // beam
            sent = unfin_idx + torch.tensor(cum_unfin)[unfin_idx]
            seen = sorted(set(zip(sent.tolist(), unfin_idx.tolist())))
            for i, sidx in enumerate(sent.tolist()):
                if len(finalized[sidx]) < beam:
                    finalized[sidx].append({"tokens": tok_clone[i], "score": eos_scores[i], "positional_scores": pos[i]})
            for us, uidx in seen:
                if not finished[us] and (len(finalized[us]) == beam or step == max_len):
                    finished[us] = True
                    finalized_sents.append(uidx)
            num_remaining -= len(finalized_sents)
        if num_remaining == 0:
            break
        assert step < max_len
        if finalized_sents:
            new_bsz = bsz - len(finalized_sents)
            batch_mask = torch.ones(bsz, dtype=torch.bool)
            batch_mask[finalized_sents] = False
            batch_idxs = torch.arange(bsz).masked_select(batch_mask)
            eos_mask, cand_beams = eos_mask[batch_idxs], cand_beams[batch_idxs]
            bbsz_offsets = bbsz_offsets[:new_bsz]
            cand_bbsz_idx = cand_beams + bbsz_offsets
            cand_scores, cand_indices = cand_scores[batch_idxs], cand_indices[batch_idxs]
            if prefix_tokens is not None:
                prefix_tokens = prefix_tokens[batch_idxs]
            orig = orig[batch_idxs]
            cands_to_ignore = cands_to_ignore[batch_idxs]
            scores = scores.view(bsz, -1)[batch_idxs].view(new_bsz * beam, -1)
            tokens = tokens.view(bsz, -1)[batch_idxs].view(new_bsz * beam, -1)
            bsz = new_bsz
        else:
            batch_idxs = None
        eos_mask[:, :beam] = ~((~cands_to_ignore) & (~eos_mask[:, :beam]))
        active_mask = eos_mask.long() * cand_size + cand_offsets[: eos_mask.size(1)]
        new_ignore, active_hypos = torch.topk(active_mask, k=beam, dim=1, largest=False)
        cands_to_ignore = new_ignore.ge(cand_size)[:, :beam]
        active_bbsz_idx = torch.gather(cand_bbsz_idx, 1, active_hypos).view(-1)
        tokens[:, : step + 1] = torch.index_select(tokens[:, : step + 1], 0, active_bbsz_idx)
        tokens.view(bsz, beam, -1)[:, :, step + 1] = torch.gather(cand_indices, 1, active_hypos)
        if step > 0:
            scores[:, :step] = torch.index_select(scores[:, :step], 0, active_bbsz_idx)
        scores.view(bsz, beam, -1)[:, :, step] = torch.gather(cand_scores, 1, active_hypos)
        reorder_state = active_bbsz_idx
    out = []
    for hyps in finalized:
        order = sorted(range(len(hyps)), key=lambda i: -float(hyps[i]["score"]))
        out.append([hyps[i] for i in order])
    return out
