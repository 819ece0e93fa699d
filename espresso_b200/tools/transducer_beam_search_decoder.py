"""Beam search for transducer models: the "adaptive expansion search" the transducer recipes decode with
(examples/asr_librispeech/run_transformer_transducer.sh:263-265: --beam 5 --transducer-expansion-beta 2
--transducer-expansion-gamma 2.3 --transducer-prefix-alpha 1), following
espresso/tools/transducer_beam_search_decoder.py:21-601 and espresso/tools/transducer_utils.py:17-757.

Per utterance and encoder frame: (1) hypotheses are sorted by length and the score of every hypothesis that is a
prefix of a longer one is merged into the longer one (prefix search, limited to `prefix_alpha` extra tokens);
(2) up to `max_num_expansions_per_step` rounds: each live hypothesis proposes its beam+beta best next symbols, those
within `expansion_gamma` of its best survive, the best beam+beta of all proposals are kept; proposals that end with
blank are set aside for the next frame, the others advance the prediction network and go on; (3) after the last round
the remaining ones pay the blank score and the best `beam` hypotheses overall move to the next frame.  Scores are
ranked normalised by the number of emissions, the final n-best by score per output token.

The search is host logic over small tensors (a handful of hypotheses); the model enters through four callbacks, which
`TransducerBeamSearchDecoder` wires to the native kernels (prediction-network step = embedding + GEMMs, joint =
LayerNorm / add+ReLU / output GEMM) exactly like the greedy decoder."""
import torch
import torch.nn.functional as F

from .. import ops as _ops
from .transducer_greedy_decoder import TransducerGreedyDecoder


class _Hyps:
    """A set of hypotheses as parallel tensors (batch dim 0): scores, seqs (pad-filled, starts with bos), lens, nemit,
    prev (last proposed symbol), hs / cs (prediction-network state [n, L, H]), dec (its output per sequence position
    [n, U, H]) and, with an LM, lm_scores, lhs / lcs, ldec."""
    PADDED = ("seqs", "dec", "ldec")

    def __init__(self, **f):
        self.f = f

    def __getattr__(self, k):
        try:
            return self.__dict__["f"][k]
        except KeyError:
            raise AttributeError(k)

    def size(self):
        return self.f["scores"].size(0)

    def take(self, index):
        """Rows `index` (a permutation / subset), padding columns beyond the longest kept sequence dropped."""
        lens = self.f["lens"].index_select(0, index)
        width = int(lens.max()) if lens.numel() else 0
        out = {}
        for k, v in self.f.items():
            if v is None:
                out[k] = None
            elif k in self.PADDED:
                out[k] = v[:, :width].index_select(0, index)
            else:
                out[k] = v.index_select(0, index)
        return _Hyps(**out)

    def where(self, mask):
        return self if bool(mask.all()) else self.take(mask.nonzero().squeeze(1))

    def repeat(self, k):
        return _Hyps(**{n: (None if v is None else v.repeat_interleave(k, dim=0)) for n, v in self.f.items()})

    @staticmethod
    def cat(a, b, pad):
        if b.size() == 0:
            return a
        if a.size() == 0:
            return b
        out = {}
        for k, v in a.f.items():
            w = b.f[k]
            if v is None:
                out[k] = None
                continue
            if k in _Hyps.PADDED:
                width = max(v.size(1), w.size(1))
                fill = pad if k == "seqs" else 0
                grow = lambda t: t if t.size(1) == width else F.pad(t, ((0, width - t.size(1)) if t.dim() == 2 else (0, 0, 0, width - t.size(1))), value=fill)  # noqa: E731
                v, w = grow(v), grow(w)
            out[k] = torch.cat((v, w), dim=0)
        return _Hyps(**out)

    def ranked(self, normalize):
        return self.f["scores"] / self.f["nemit"] if normalize else self.f["scores"]

    def sort_by_score(self, normalize, descending=True):
        return self if self.size() == 0 else self.take(self.ranked(normalize).argsort(descending=descending))

    def top_k(self, k, normalize):
        if k > self.size():
            return self.sort_by_score(normalize)
        return self.take(torch.topk(self.ranked(normalize), k, largest=True, sorted=True)[1])

    def last(self, key):
        v = self.f[key]
        idx = (self.f["lens"] - 1).view(-1, 1, 1).expand(-1, 1, v.size(2))
        return v.gather(1, idx).squeeze(1)

    def set_last_(self, key, value):
        v = self.f[key]
        idx = (self.f["lens"] - 1).view(-1, 1, 1).expand(-1, 1, v.size(2))
        v.scatter_(1, idx, value.unsqueeze(1).to(v.dtype))

    def append_(self, tokens, blank, pad):
        """Record the proposed symbols: non-blank ones extend their sequence (Hypotheses.append_tokens_)."""
        self.f["prev"] = tokens.clone()
        is_blank = tokens == blank
        if bool(is_blank.all()):
            return  # (the reference leaves the emission counters untouched in this case)
        lens = self.f["lens"]
        if bool((tokens[lens == lens.max()] != blank).any()):
            self.f["seqs"] = F.pad(self.f["seqs"], (0, 1), value=pad)
            for k in ("dec", "ldec"):
                if self.f.get(k) is not None:
                    self.f[k] = F.pad(self.f[k], (0, 0, 0, 1))
        self.f["seqs"].scatter_(1, lens.unsqueeze(1), tokens.masked_fill(is_blank, pad).unsqueeze(1))
        self.f["lens"] = lens + (~is_blank).long()
        self.f["nemit"] = self.f["nemit"] + 1


class AdaptiveExpansionSearch:
    """Model-agnostic search.  Callbacks:
         pred_step(prev [n] int64, hs, cs) -> (out [n, H], hs, cs)          prediction network, one step
         joint_lprobs(frame, out [n, H]) -> fp32 [n, V]                     log-probs of the joint at encoder frame `frame`
         lm_step(prev [n], lhs, lcs) -> (feat [n, H'], lhs, lcs)            LM, one step (optional)
         lm_lprobs(feat [n, H']) -> fp32 [n, V_lm]                          LM log-probs (optional)
       `init_state(n)` / `lm_init_state(n)` return zero states (hs, cs) with batch dim 0."""

    def __init__(self, vocab_size, blank, pad, eos, bos, beam_size, max_num_expansions_per_step=2, expansion_beta=0,
                 expansion_gamma=None, prefix_alpha=None, normalize_scores=True, model_predicts_eos=False, lm_weight=1.0,
                 no_blank_in_lm=False):
        self.V, self.blank, self.pad, self.eos, self.bos = vocab_size, blank, pad, eos, bos
        self.beam = min(beam_size, vocab_size - (1 if pad != blank else 0))
        self.E, self.beta, self.gamma, self.alpha = max_num_expansions_per_step, expansion_beta, expansion_gamma, prefix_alpha
        assert self.E > 0 and expansion_beta >= 0 and (expansion_gamma is None or expansion_gamma > 0.0)
        assert prefix_alpha is None or prefix_alpha > 0
        self.normalize, self.predicts_eos = normalize_scores, model_predicts_eos
        self.lm_weight, self.no_blank_in_lm = lm_weight, no_blank_in_lm

    # ---- LM fusion over the non-blank symbols, transducer's blank / non-blank split preserved -------------------
    def _fuse(self, lp, lm_lp):
        nb = self._nonblank.to(lp.device)
        if not self.no_blank_in_lm:
            lm_lp = lm_lp[:, nb]
        lp_nb = lp[:, nb]
        fused = lp_nb + self.lm_weight * lm_lp
        scale = lp_nb.exp().sum(1).log() - fused.exp().sum(1).log()
        lp = lp.clone()
        lp[:, nb] = fused + scale[:, None]
        padded = torch.cat((lm_lp[:, : self.blank], lm_lp.new_zeros(lm_lp.size(0), 1), lm_lp[:, self.blank:]), dim=1)
        return lp, padded, scale

    def _lm_token(self, tok):
        return torch.where(tok > self.blank, tok - 1, tok) if self.no_blank_in_lm else tok

    def search(self, n_frames, cb, device, bos_token=None, use_lm=False):
        """One utterance.  Returns (sequences int64 [n, U] without the leading bos, scores [n]) sorted best first."""
        self._nonblank = torch.ones(self.V, dtype=torch.bool)
        self._nonblank[self.blank] = False
        prev = torch.full((1,), self.bos if bos_token is None else bos_token, dtype=torch.long, device=device)
        hs, cs = cb["init_state"](1)
        out, hs, cs = cb["pred_step"](prev, hs, cs)
        f = dict(scores=torch.zeros(1, device=device), seqs=prev.unsqueeze(1).clone(), lens=torch.ones(1, dtype=torch.long, device=device),
                 nemit=torch.zeros(1, dtype=torch.long, device=device), prev=prev, hs=hs, cs=cs, dec=out.unsqueeze(1).clone(),
                 lm_scores=None, lhs=None, lcs=None, ldec=None)
        if use_lm:
            lhs, lcs = cb["lm_init_state"](1)
            lfeat, lhs, lcs = cb["lm_step"](self._lm_token(prev), lhs, lcs)
            f.update(lm_scores=torch.zeros(1, device=device), lhs=lhs, lcs=lcs, ldec=lfeat.unsqueeze(1).clone())
        nxt = _Hyps(**f)
        for t in range(n_frames):
            nxt = nxt.take(nxt.lens.argsort(descending=True))
            hyps = self._prefix_merge(nxt, t, cb, use_lm)
            set_aside = None
            for e in range(self.E):
                lp = cb["joint_lprobs"](t, hyps.last("dec"))
                lm_padded = None
                if use_lm:
                    lp, lm_padded, _ = self._fuse(lp, cb["lm_lprobs"](hyps.last("ldec")))
                if self.predicts_eos:
                    lp[:, self.blank] = torch.logaddexp(lp[:, self.blank], lp[:, self.eos])
                    lp[:, self.eos] = float("-inf")
                cand = self._expand(hyps, lp, lm_padded)
                is_blank = cand.prev == self.blank
                blanks = cand.where(is_blank)
                set_aside = blanks if e == 0 else _Hyps.cat(set_aside, blanks, self.pad)
                live = cand.where(~is_blank)
                if live.size() == 0:
                    nxt = set_aside.top_k(self.beam, self.normalize)
                    break
                out, live.f["hs"], live.f["cs"] = cb["pred_step"](live.prev, live.hs, live.cs)
                live.set_last_("dec", out)
                if use_lm:
                    lfeat, live.f["lhs"], live.f["lcs"] = cb["lm_step"](self._lm_token(live.prev), live.lhs, live.lcs)
                    live.set_last_("ldec", lfeat)
                if e < self.E - 1:
                    hyps = live
                else:  # out of expansion rounds: the survivors take the blank of this frame
                    lp = cb["joint_lprobs"](t, out)
                    live.f["scores"] = live.scores + lp[:, self.blank]
                    live.f["prev"] = torch.full_like(live.prev, self.blank)
                    live.f["nemit"] = live.nemit + 1
                    nxt = _Hyps.cat(set_aside, live, self.pad).top_k(self.beam, self.normalize)
        nxt.f["scores"] = nxt.scores / (nxt.lens - 1)
        nxt = nxt.sort_by_score(False)
        return nxt.seqs[:, 1:], nxt.scores

    def _expand(self, hyps, lp, lm_padded):
        """Each hypothesis proposes its k best symbols; prune by value; keep the k best proposals (select_k_expansions)."""
        tot = lp + hyps.scores.unsqueeze(-1)
        k = min(self.beam + self.beta, tot.size(1) - (1 if self.pad != self.blank else 0))
        scores, idx = torch.topk(tot, k=k)
        cand = hyps.repeat(k)
        cand.f["scores"] = scores.reshape(-1)
        if lm_padded is not None:
            cand.f["lm_scores"] = cand.lm_scores + lm_padded.gather(1, idx).reshape(-1)
        cand.append_(idx.reshape(-1), self.blank, self.pad)
        if self.gamma is not None:
            keep = scores >= (scores[:, :1] - self.gamma)
            if not bool(keep.all()):
                cand = cand.where(keep.reshape(-1))
        return cand.top_k(k, self.normalize)

    def _prefix_merge(self, hyps, t, cb, use_lm):
        """hyps sorted by non-increasing length.  If hypothesis i is a prefix of the longer j (at most alpha tokens
        longer), the probability of reaching j's sequence from i within this frame is added to j's score."""
        n = hyps.size()
        lens = hyps.lens
        seqs = hyps.seqs
        rel = torch.zeros(n, n, dtype=torch.bool)
        for j in range(n - 1):
            for i in range(j + 1, n):
                li = int(lens[i])
                rel[i, j] = bool(lens[i] < lens[j]) and bool((seqs[i, :li] == seqs[j, :li]).all())
        if self.alpha is not None:
            rel = rel & (lens.cpu().unsqueeze(1) + self.alpha >= lens.cpu().unsqueeze(0))
        if not bool(rel.any()):
            return hyps
        for j in range(n - 1):
            for i in range(j + 1, n):
                if not bool(rel[i, j]):
                    continue
                li, lj = int(lens[i]), int(lens[j])
                # positions li-1 (in i's history) then li .. lj-2 (in j's): each emits j's next token
                steps = [(i, li - 1)] + [(j, k) for k in range(li, lj - 1)]
                score = hyps.scores[i].clone()
                lm_score = hyps.lm_scores[i].clone() if use_lm else None
                for (row, pos) in steps:
                    lp = cb["joint_lprobs"](t, hyps.dec[row: row + 1, pos])[0]
                    tok = int(seqs[j, pos + 1])
                    score = score + lp[tok]
                    if use_lm:
                        lm_lp = cb["lm_lprobs"](hyps.ldec[row: row + 1, pos])[0]
                        lt = tok - 1 if (self.no_blank_in_lm and tok > self.blank) else tok
                        lm_score = lm_score + lm_lp[lt]
                        _, _, scale = self._fuse(lp.unsqueeze(0), lm_lp.unsqueeze(0))
                        score = score + self.lm_weight * lm_lp[lt] + scale[0]
                hyps.f["scores"][j] = torch.logaddexp(hyps.scores[j], score)
                if use_lm:
                    hyps.f["lm_scores"][j] = torch.logaddexp(hyps.lm_scores[j], lm_score)
        return hyps


def beam_state(B, K, beam, E, alpha, pool, n_frames, device):
    """The device search's tables (flat, utterance-major; include/espresso_b200.h: EspRnntBeam):
         rows      score, nemit, len, node (prefix-pool node), srow (state row of this round), fsrc (state reference
                   (round * B*K + row) a row takes at the end of the frame), parent / prev (state row and token the
                   predictor advances) -- K = beam + beta rows per utterance; nrow (rows), nlive (rows in the round)
         set-aside a_score, a_nemit, a_len, a_node, a_src -- E * K per utterance; na
         pool      p_parent, p_tok, p_len, p_hash (64-bit rolling prefix hash) -- `pool` nodes per utterance; npool
         merge     m_pair (j, i, first step, steps) x beam (beam - 1) / 2, m_ring / m_tok per path step; m_npair
       Every utterance starts with one row: the root node (bos), score 0."""
    BK, A, Pm = B * K, E * K, beam * (beam - 1) // 2
    i32 = dict(dtype=torch.int32, device=device)
    st = dict(B=B, K=K, E=E, A=A, P=pool, Pm=Pm, S=max(Pm * alpha, 1), alpha=alpha, ring_stride=(E + 1) * BK)
    st.update(score=torch.zeros(BK, dtype=torch.float32, device=device), nemit=torch.zeros(BK, **i32),
              len=torch.ones(BK, **i32), node=torch.zeros(BK, **i32), srow=torch.arange(BK, **i32), fsrc=torch.arange(BK, **i32),
              parent=torch.arange(BK, **i32), prev=torch.zeros(BK, **i32), nrow=torch.ones(B, **i32),
              nlive=torch.zeros(B, **i32), nframes=n_frames.to(device=device, dtype=torch.int32).contiguous(),
              a_score=torch.zeros(B * A, dtype=torch.float32, device=device), a_nemit=torch.zeros(B * A, **i32),
              a_len=torch.zeros(B * A, **i32), a_node=torch.zeros(B * A, **i32), a_src=torch.zeros(B * A, **i32),
              na=torch.zeros(B, **i32), p_parent=torch.full((B * pool,), -1, **i32), p_tok=torch.zeros(B * pool, **i32),
              p_len=torch.ones(B * pool, **i32), p_hash=torch.zeros(B * pool, dtype=torch.int64, device=device),
              npool=torch.ones(B, **i32), m_pair=torch.zeros(B * max(Pm, 1) * 4, **i32), m_ring=torch.zeros(B * st["S"], **i32),
              m_tok=torch.zeros(B * st["S"], **i32), m_npair=torch.zeros(B, **i32))
    return st


class BatchedAdaptiveExpansionSearch:
    """The adaptive expansion search for a whole batch, its steps as native kernels (csrc/transducer_beam.cu): per frame
    one prefix merge (rnnt_beam_prefix_merge, the joint over the listed path steps, rnnt_beam_merge_scores), then up to
    E rounds of joint over all rows, rnnt_beam_lprobs, rnnt_beam_select, state gather, predictor (and LM) step.  Gives
    every utterance the n-best AdaptiveExpansionSearch gives it (same parameters; prefix_alpha must be set).

    Hypotheses are rows of fixed tables (beam_state); a row's history is a node of a per-utterance prefix pool, its
    decoder state the predictor / LM state plus a ring of its last `prefix_alpha` joint-space projections (and LM output
    features).  States live in per-round buffers [E + 1, B*K, ...]: round e reads buffer e, its predictor step writes
    buffer e + 1, and the frame's survivors are gathered back into buffer 0 by their (round, row) references, so a blank
    set aside in round e needs no copy.  Rows of utterances that are done (or outside their frames) are carried
    through the fixed-shape steps and ignored.  The only host sync per round is the "any live row left" read.

    Callbacks (n rows, batch dim 0):
         init_state(n) -> (hs, cs)                   lm_init_state(n) -> (lhs, lcs)      zero states
         pred_step(prev [n] int64, hs, cs) -> (out [n, H], hs, cs)
         project(out) -> pd [n, J]                                                       joint-space projection
         joint_logits(frame [n] int32, pd) -> logits [n, >= V]   frame = b * T + t (the utterance's encoder frame)
         lm_step(prev [n], lhs, lcs) -> (feat [n, H'], lhs, lcs)  lm_logits(feat) -> logits [n, >= V_lm]"""

    def __init__(self, core, temperature=1.0):
        assert core.alpha is not None, "the batched search needs prefix_alpha"
        self.c, self.temperature = core, temperature
        self.K = min(core.beam + core.beta, core.V - (1 if core.pad != core.blank else 0))

    def search(self, n_frames, T, cb, device, bos_token=None, use_lm=False):
        """n_frames int [B] (frames each utterance decodes), T the frame stride of `frame`.  Returns per utterance
        (sequences int64 [n, U] without the leading bos, pad-filled, scores fp32 [n]) sorted best first."""
        c, K, E, alpha = self.c, self.K, self.c.E, self.c.alpha
        B = int(n_frames.numel())
        BK = B * K
        t_max = int(n_frames.max()) if B else 0
        st = beam_state(B, K, c.beam, E, alpha, 1 + t_max * E * K, n_frames, device)
        bos = c.bos if bos_token is None else bos_token
        st["p_tok"][::st["P"]] = bos
        lm_kw = dict(lm_weight=c.lm_weight, no_blank_in_lm=c.no_blank_in_lm) if use_lm else {}

        # per-round state buffers [E + 1, B*K, ...]; rings [alpha, E + 1, B*K, .] (age 0 = the newest output)
        prev = torch.full((BK,), bos, dtype=torch.long, device=device)
        out, hs, cs = cb["pred_step"](prev, *cb["init_state"](BK))
        bufs = {"hs": hs, "cs": cs}
        pd = cb["project"](out)
        rings = {"pd": pd}
        if use_lm:
            feat, lhs, lcs = cb["lm_step"](c._lm_token(prev), *cb["lm_init_state"](BK))
            bufs.update(lhs=lhs, lcs=lcs)
            rings["lm"] = feat
        for k, v in list(bufs.items()):
            bufs[k] = v.new_zeros((E + 1,) + tuple(v.shape))
            bufs[k][0] = v
        for k, v in list(rings.items()):
            rings[k] = v.new_zeros((alpha, E + 1) + tuple(v.shape))
            rings[k][0, 0] = v
        row_frame = (torch.arange(BK, device=device, dtype=torch.int32) // K) * T
        step_frame = (torch.arange(B * st["S"], device=device, dtype=torch.int32) // st["S"]) * T
        flag = torch.empty(B, dtype=torch.int32, pin_memory=device.type == "cuda")

        def any_live():
            flag.copy_(st["nlive"], non_blocking=True)
            if device.type == "cuda":
                torch.cuda.current_stream(device).synchronize()
            return bool(flag.any())

        def advance(e):  # the live rows' predictor (and LM) step from their parents' states: buffer e -> e + 1
            par = st["parent"]
            g = {k: _ops.gather_rows(v[e].reshape(BK, -1), par).view(v[e].shape) for k, v in bufs.items()}
            tok = st["prev"].long()
            o, bufs["hs"][e + 1], bufs["cs"][e + 1] = cb["pred_step"](tok, g["hs"], g["cs"])
            newest = {"pd": cb["project"](o)}
            if use_lm:
                newest["lm"], bufs["lhs"][e + 1], bufs["lcs"][e + 1] = cb["lm_step"](c._lm_token(tok), g["lhs"], g["lcs"])
            for k, r in rings.items():
                r[0, e + 1] = newest[k]
                for a in range(alpha - 1):
                    _ops.gather_rows(r[a, e], par, out=r[a + 1, e + 1])

        def lm_logits_rows(rows):
            return cb["lm_logits"](rows) if use_lm else None

        for t in range(t_max):
            _ops.rnnt_beam_prefix_merge(st, t, alpha)
            if st["Pm"] > 0:
                idx = st["m_ring"]
                lg = cb["joint_logits"](step_frame + t, _ops.gather_rows(rings["pd"].reshape(-1, rings["pd"].shape[-1]), idx))
                lml = lm_logits_rows(_ops.gather_rows(rings["lm"].reshape(-1, rings["lm"].shape[-1]), idx)) if use_lm else None
                _ops.rnnt_beam_merge_scores(lg, c.V, st, self.temperature, c.blank, lml, **lm_kw)
            for e in range(E):
                cur = _ops.gather_rows(rings["pd"][0, 0], st["srow"]) if e == 0 else rings["pd"][0, e]
                lm_cur = None
                if use_lm:
                    lm_cur = lm_logits_rows(_ops.gather_rows(rings["lm"][0, 0], st["srow"]) if e == 0 else rings["lm"][0, e])
                val, tok, lpb = _ops.rnnt_beam_lprobs(cb["joint_logits"](row_frame + t, cur), c.V, st["score"], K, c.blank,
                                                      self.temperature, c.eos, c.predicts_eos, lm_cur, **lm_kw)
                _ops.rnnt_beam_select(val, tok, lpb, st, e, c.beam, c.blank, c.gamma, c.normalize, False)
                if not any_live():
                    break
                advance(e)
                if e == E - 1:  # out of expansion rounds: the survivors take the blank of this frame
                    _, _, lpb = _ops.rnnt_beam_lprobs(cb["joint_logits"](row_frame + t, rings["pd"][0, E]), c.V, st["score"], 1,
                                                      c.blank, self.temperature)
                    _ops.rnnt_beam_select(val, tok, lpb, st, e, c.beam, c.blank, c.gamma, c.normalize, True)
            for v in list(bufs.values()) + [r[a] for r in rings.values() for a in range(alpha)]:
                v[0].copy_(_ops.gather_rows(v.reshape((E + 1) * BK, -1), st["fsrc"]).view(v[0].shape))
        tokens, scores, lens = _ops.rnnt_beam_finalize(st, c.pad)
        nrow, lens = st["nrow"].tolist(), lens.cpu()
        return [(tokens[b, :nrow[b], :int(lens[b, :nrow[b]].max())], scores[b, :nrow[b]]) for b in range(B)]


class TransducerBeamSearchDecoder(TransducerGreedyDecoder):
    """The reference's constructor arguments (transducer_beam_search_decoder.py:22-42); decode() returns the 1-best like
    the reference (tokens [B, U] padded, scores [B], None), generate() the n-best lists."""

    def __init__(self, models, dictionary, beam_size=1, max_len=0, max_num_expansions_per_step=2, expansion_beta=0,
                 expansion_gamma=None, prefix_alpha=None, normalize_scores=True, temperature=1.0, eos=None, bos=None, blank=None,
                 pad=None, model_predicts_eos=False, symbols_to_strip_from_output=None, lm_model=None, lm_weight=1.0, **unused):
        super().__init__(models, dictionary, max_len=max_len, max_num_expansions_per_step=max_num_expansions_per_step,
                         temperature=temperature, eos=eos, bos=bos, blank=blank, model_predicts_eos=model_predicts_eos,
                         symbols_to_strip_from_output=symbols_to_strip_from_output, lm_model=lm_model, lm_weight=lm_weight)
        if pad is not None:
            self.pad = pad
        self.core = AdaptiveExpansionSearch(self.vocab_size, self.blank, self.pad, self.eos, self.bos, beam_size,
                                            max_num_expansions_per_step, expansion_beta, expansion_gamma, prefix_alpha,
                                            normalize_scores, model_predicts_eos, lm_weight, self.no_blank_in_lm)

    @torch.no_grad()
    def _generate(self, sample, bos_token=None):
        m = self.model
        m.eval()
        enc_out = m.forward_encoder(sample["net_input"])
        enc = enc_out["b200_out"]
        enc_lens = enc_out["src_lengths"][0].cpu().tolist()
        B, T, d = enc.shape
        pe_all = m.project(enc.reshape(B * T, d), "encoder")[0].view(B, T, -1)
        W = m.fc_out_weight()[0]
        # The batched search's steps are CUDA kernels.  The per-utterance host search stays the path for alpha unset and
        # for CPU tensors, where ops is replaced by its plain-PyTorch statement (the product's ops refuse CPU tensors).
        batched = self.core.alpha is not None and enc.is_cuda
        search = self._generate_batched if batched else self._generate_host
        return search(m, pe_all, W, enc_lens, T, enc.device, bos_token)

    def _generate_host(self, m, pe_all, W, enc_lens, T, dev, bos_token):
        """One AdaptiveExpansionSearch per utterance."""
        B = pe_all.size(0)
        V = self.vocab_size
        nl = len(m.decoder.layers)
        hid = m.decoder.layers[0].weight_hh.shape[1]
        lm = self.lm_model
        results = []
        for b in range(B):
            def pred_step(prev, hs, cs):
                top, nh, nc = self._predictor_step(prev, [hs[:, i] for i in range(nl)], [cs[:, i] for i in range(nl)])
                return top, torch.stack(nh, dim=1), torch.stack(nc, dim=1)

            def joint_lprobs(t, out, _b=b):
                pd = m.project(out, "decoder")[0]
                logits, _ = m.joint_logits(pe_all[_b, t].contiguous().view(1, 1, -1), pd.view(1, out.size(0), -1), W)
                return torch.log_softmax(logits[:, :V].float() / self.temperature, dim=-1)

            cb = dict(pred_step=pred_step, joint_lprobs=joint_lprobs,
                      init_state=lambda n: (torch.zeros(n, nl, hid, dtype=torch.bfloat16, device=dev),
                                            torch.zeros(n, nl, hid, dtype=torch.float32, device=dev)))
            if lm is not None:
                lm.eval()
                ld = lm.decoder
                lnl, lh = len(ld.layers), ld.hidden_size
                w = ld.embed_tokens.weight

                def lm_step(prev, lhs, lcs):
                    y, nh, nc, _ = ld.step(ld.embed_tokens(prev), [lhs[:, i] for i in range(lnl)], [lcs[:, i] for i in range(lnl)], None)
                    return y, torch.stack(nh, dim=1), torch.stack(nc, dim=1)

                cb.update(lm_step=lm_step, lm_lprobs=lambda feat: torch.log_softmax(ld.output_layer(feat.to(w.dtype)).float(), dim=-1),
                          lm_init_state=lambda n: (w.new_zeros(n, lnl, lh), w.new_zeros(n, lnl, lh)))
            n_frames = min(enc_lens[b], self.max_len) if self.max_len > 0 else enc_lens[b]
            results.append(self.core.search(n_frames, cb, dev, bos_token=bos_token, use_lm=lm is not None))
        return results

    def _generate_batched(self, m, pe_all, W, enc_lens, T, dev, bos_token):
        """The whole batch in one BatchedAdaptiveExpansionSearch."""
        B, _, J = pe_all.shape
        V = self.vocab_size
        nl = len(m.decoder.layers)
        hid = m.decoder.layers[0].weight_hh.shape[1]
        pe_rows = pe_all.reshape(B * T, J).contiguous()

        def pred_step(prev, hs, cs):
            top, nh, nc = self._predictor_step(prev, [hs[:, i] for i in range(nl)], [cs[:, i] for i in range(nl)])
            return top, torch.stack(nh, dim=1), torch.stack(nc, dim=1)

        def joint_logits(frame, pd):
            n = pd.size(0)
            return m.joint_logits(_ops.gather_rows(pe_rows, frame).view(n, 1, J), pd.contiguous().view(n, 1, J), W)[0]

        cb = dict(pred_step=pred_step, project=lambda out: m.project(out, "decoder")[0], joint_logits=joint_logits,
                  init_state=lambda n: (torch.zeros(n, nl, hid, dtype=torch.bfloat16, device=dev),
                                        torch.zeros(n, nl, hid, dtype=torch.float32, device=dev)))
        lm = self.lm_model
        if lm is not None:
            lm.eval()
            ld = lm.decoder
            lnl, lh = len(ld.layers), ld.hidden_size
            w = ld.embed_tokens.weight

            def lm_step(prev, lhs, lcs):
                y, nh, nc, _ = ld.step(ld.embed_tokens(prev), [lhs[:, i] for i in range(lnl)], [lcs[:, i] for i in range(lnl)], None)
                return y, torch.stack(nh, dim=1), torch.stack(nc, dim=1)

            cb.update(lm_step=lm_step, lm_logits=lambda feat: ld.output_layer(feat.to(w.dtype).contiguous()),
                      lm_init_state=lambda n: (w.new_zeros(n, lnl, lh), w.new_zeros(n, lnl, lh)))
        n_frames = torch.tensor([min(n, self.max_len) if self.max_len > 0 else n for n in enc_lens], dtype=torch.int32)
        search = BatchedAdaptiveExpansionSearch(self.core, self.temperature)
        return search.search(n_frames, T, cb, dev, bos_token=bos_token, use_lm=lm is not None)

    @torch.no_grad()
    def decode(self, models, sample, bos_token=None, **unused):
        res = self._generate(sample, bos_token)
        width = max(max(int((s[0] != self.pad).sum()) for s, _ in res), 1)
        tokens = torch.full((len(res), width), self.pad, dtype=torch.long, device=res[0][0].device)
        for b, (s, _) in enumerate(res):
            row = s[0][s[0] != self.pad]
            tokens[b, : row.numel()] = row
        return tokens, torch.stack([sc[0] for _, sc in res]), None

    def generate(self, models, sample, bos_token=None, **unused):
        strip = sorted(self.symbols_to_strip_from_output | {self.pad})
        out = []
        for seqs, scores in self._generate(sample, bos_token):
            st = torch.tensor(strip, device=seqs.device)
            out.append([{"tokens": seqs[k][~torch.isin(seqs[k], st)], "score": scores[k], "attention": None, "alignment": None,
                         "positional_scores": None} for k in range(seqs.size(0))])
        return out
