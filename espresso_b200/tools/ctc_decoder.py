"""CTC decoding (espresso/tools/ctc_decoder.py:18-188).

Greedy (beam_size 1, no LM; also what validation uses): argmax over the vocabulary per frame, collapse repeats
(unique_consecutive), drop blanks.  The argmax runs in esp_argmax_rows; the collapse is a tiny host loop over B sequences.

Beam search (beam_size > 1 or an LM): a frame-synchronous CTC prefix beam search on the device (esp_ctc_beam_frames /
_search / _finalize, include/espresso_b200.h), optionally fused with a subword language model (shallow fusion): the
recipes' LSTM LM (`lstm_lm_espresso`) or a Transformer LM (`transformer_lm`).  The search kernel launches once for all
frames without an LM and once per frame with one; between frames the LM rows follow the search's new_order and step on
the tokens appended in that frame, rows without a new token keep their state.  The LSTM's (h, c) rows are re-gathered;
the Transformer LM keeps a KV cache indexed by frame slot and a path table per hypothesis (IncrementalDecoder's
prefix-state mode), so prefixes of different lengths share one cache and nothing in it moves.  An LM vocabulary one
symbol short of the CTC vocabulary is the CTC vocabulary without the blank.  The host reads the results once per
batch, after finalize.

The reference reaches its beam path through flashlight's Lexicon(Free)Decoder with a KenLM model; its defaults carry
over: beam_size_token = min(beam, V), beam_threshold = min(beam, V), unk excluded.  An ARPA n-gram LM
(models.ngram_lm.NgramLanguageModel) is scored inside the search kernel (esp_ctc_ngram_search / _finalize), so its
search is one launch for all frames as without an LM.  Without a lexicon its vocabulary is the dictionary's symbols and
`word_score` is a bonus per emitted token; with `lexicon` (flashlight's lexicon file) the search follows the lexicon
trie, the n-gram scores whole words and `word_score` is a bonus per word (unk_weight = -inf, no silence token).  Scores
of the n-gram are log10, as KenLM's.  A KenLM path (load the ARPA with NgramLanguageModel.from_arpa instead), a
lexicon without an n-gram LM (so also with a Transformer or LSTM LM) and LMs other than these (word LMs, the look-ahead
and multi-level word LMs) are refused with NotImplementedError.

decode(models, sample) -> (tokens int64 [B, U] padded, scores, alignments) like the reference's `decode` (:80-98);
generate() -> per sentence a list of up to `nbest` dicts (tokens, score in natural log, alignment).  A sentence without a
hypothesis (through a lexicon: its last beam ends inside words only) gets one empty hypothesis with score -inf, so that
callers such as recognize() still emit and score it."""
import math

import torch

from .. import ops as _ops


class CTCDecoder:
    def __init__(self, dictionary, blank_idx=None, pad_idx=None, beam_size=1, lm_model=None, lm_weight=0.0, word_score=0.0,
                 print_alignment=False, lexicon=None, beam_size_token=None, beam_threshold=None, nbest=1, allow_unk=False):
        self.pad = dictionary.pad() if pad_idx is None else pad_idx
        self.blank = dictionary.index("<s>") if blank_idx is None else blank_idx
        self.beam_size = int(beam_size)
        self.greedy = self.beam_size == 1 and lm_model is None
        self.eos = dictionary.eos() if hasattr(dictionary, "eos") else None
        self.unk = dictionary.unk() if hasattr(dictionary, "unk") else None
        from ..models.ngram_lm import LexiconTrie, NgramLanguageModel

        if isinstance(lm_model, str):
            raise NotImplementedError("KenLM model paths are not read; load the ARPA file with "
                                      "NgramLanguageModel.from_arpa(path) and pass the model")
        self.ngram = isinstance(lm_model, NgramLanguageModel)
        if lexicon is not None and not self.ngram:
            raise NotImplementedError("lexicon-constrained CTC decoding needs an n-gram LM (NgramLanguageModel.from_arpa)")
        self.lm_model, self.lm_weight, self.word_score = lm_model, float(lm_weight or 0.0), float(word_score)
        self.lm_blank = -1
        self.transformer = False
        self.lexicon, self._tok_word, self._tok_word_dev = None, None, {}
        if self.ngram:
            if lexicon is not None:
                self.lexicon = lexicon if isinstance(lexicon, LexiconTrie) else LexiconTrie.from_file(lexicon, dictionary, lm_model)
            else:  # the n-gram's words are the dictionary's symbols; others (and the blank) are <unk>
                self._tok_word = torch.tensor([lm_model.index(dictionary[i]) for i in range(len(dictionary))], dtype=torch.int32)
        elif lm_model is not None:
            from ..models.lstm_lm import LSTMLanguageModelEspresso
            from ..models.transformer_lm import TransformerLanguageModel

            self.transformer = isinstance(lm_model, TransformerLanguageModel)
            if not (self.transformer or isinstance(lm_model, LSTMLanguageModelEspresso)) or getattr(lm_model, "is_wordlm", False):
                raise NotImplementedError(
                    "CTC LM fusion supports the LSTM subword LM (lstm_lm_espresso), the Transformer subword LM "
                    "(transformer_lm) and ARPA n-grams only, not %s: word, look-ahead and multi-level LMs advance on whole "
                    "words" % type(lm_model).__name__)
            if self.transformer and lm_model.engine is None:
                # its prefix steps run on the native engine that finalize_ builds (flat bf16 parameters on the device)
                raise NotImplementedError("CTC fusion runs a TransformerLanguageModel on its native engine only; call "
                                          "finalize_(device) on the LM before building the decoder")
            n_lm, V = lm_model.decoder.embed_tokens.num_embeddings, len(dictionary)
            if n_lm not in (V, V - 1):
                raise ValueError("LM vocabulary (%d) does not match the CTC dictionary (%d)" % (n_lm, V))
            # an LM vocabulary one symbol short = the CTC vocabulary without the blank (as for transducers)
            self.lm_blank = self.blank if n_lm == V - 1 else -1
        self.nbest = int(nbest)
        self.beam_size_token = beam_size_token
        self.beam_threshold = beam_threshold
        self.allow_unk = allow_unk
        self.print_alignment = print_alignment

    @torch.no_grad()
    def decode(self, models, sample, **unused):
        model = models[0]
        model.eval()
        net = model(**sample["net_input"])
        out = net["b200_out"]  # [B, T', ld]
        V = net["encoder_out"][0].size(-1)
        if self.greedy:
            return self._greedy(out, V, net["src_lengths"][0].tolist())
        tokens, lens, scores, frames = self.search(out, V, net["src_lengths"][0])
        U = max(int(lens[:, 0].max()) if lens.numel() else 0, 1)
        best = tokens[:, 0, :U].long()
        return best, scores[:, 0], (frames[:, 0, :U].long() if frames is not None else None)

    def _greedy(self, out, V, lens):
        B, T, ld = out.shape
        am = _ops.argmax_rows(out.reshape(B * T, ld), V).view(B, T).cpu()
        hyps = []
        for b in range(B):
            seq = am[b, : lens[b]]
            if seq.numel():
                keep = torch.ones_like(seq, dtype=torch.bool)
                keep[1:] = seq[1:] != seq[:-1]          # unique_consecutive
                seq = seq[keep]
                seq = seq[seq != self.blank]
            hyps.append(seq.long())
        U = max([h.numel() for h in hyps] + [1])
        tokens = torch.full((B, U), self.pad, dtype=torch.long)
        for b, h in enumerate(hyps):
            tokens[b, : h.numel()] = h
        return tokens, None, None

    @torch.no_grad()
    def search(self, logits, V, in_lens):
        """Prefix beam search over logits bf16 [B, T', ld] -> host tensors (tokens [B, nbest, T'] pad-filled, lengths
        [B, nbest], scores [B, nbest] (natural log, -inf for missing hypotheses), frames [B, nbest, T'] or None)."""
        B, T, _ = logits.shape
        dev = logits.device
        beam = self.beam_size
        K = self.beam_size_token if self.beam_size_token is not None else min(beam, V)
        thr = self.beam_threshold if self.beam_threshold is not None else float(min(beam, V))
        lens = in_lens.to(device=dev, dtype=torch.int32)
        frames = _ops.ctc_beam_frames(logits, V, lens, K, self.blank, self.pad, self.eos, -1 if self.allow_unk else self.unk)
        lm = self.lm_model
        lm_kw = {}
        if self.ngram:
            ws = _ops.ctc_ngram_workspace(B, T, beam, dev)
            tw = None
            if self.lexicon is None:
                tw = self._tok_word_dev.get(str(dev))
                if tw is None:
                    tw = self._tok_word_dev[str(dev)] = self._tok_word.to(dev)
            _ops.ctc_ngram_search(logits, V, lens, frames, beam, thr, ws, lm, tok_word=tw, lexicon=self.lexicon,
                                  lm_weight=self.lm_weight, word_score=self.word_score)
            res = _ops.ctc_ngram_finalize(lens, T, V, beam, self.nbest, ws, lm, lexicon=self.lexicon, lm_weight=self.lm_weight,
                                          pad=self.pad, want_frames=self.print_alignment)
            return tuple(r.cpu() if r is not None else None for r in res)
        ws = _ops.ctc_beam_workspace(B, T, beam, dev)
        if lm is None:
            _ops.ctc_beam_search(logits, V, lens, frames, beam, thr, 0, T, ws, word_score=self.word_score, eos=self.eos)
        elif self.transformer:
            lm.eval()
            N = B * beam
            eos_lm = self.eos - 1 if (self.lm_blank >= 0 and self.eos > self.lm_blank) else self.eos
            lm_kw = dict(V_lm=lm.decoder.embed_tokens.num_embeddings, lm_blank=self.lm_blank, lm_weight=self.lm_weight)
            # slot 0: every row feeds the eos context into an empty prefix; slot t + 1: frame t's tokens
            state = lm.init_prefix_state(B, beam, T)
            rows_ix = torch.arange(N, dtype=torch.int32, device=dev)
            rows = lm.prefix_step(0, torch.full((N,), eos_lm, dtype=torch.int32, device=dev), torch.ones_like(rows_ix), rows_ix,
                                  state)
            for t in range(T):
                new_order, grown, fed = _ops.ctc_beam_search(logits, V, lens, frames, beam, thr, t, t + 1, ws, lm=rows,
                                                             word_score=self.word_score, eos=self.eos, want_order=True, **lm_kw)
                new_rows = lm.prefix_step(t + 1, fed, grown, new_order, state)
                rows = torch.where(grown.view(N, 1) != 0, new_rows, rows.index_select(0, new_order.long()))
            if T == 0:  # no frame to search: just the initial state
                _ops.ctc_beam_search(logits, V, lens, frames, beam, thr, 0, 0, ws, lm=rows, word_score=self.word_score,
                                     eos=self.eos, **lm_kw)
            lm_kw["lm"] = rows
        else:
            lm.eval()
            N = B * beam
            n_lm = lm.decoder.embed_tokens.num_embeddings
            eos_lm = self.eos - 1 if (self.lm_blank >= 0 and self.eos > self.lm_blank) else self.eos
            # the LM starts from its eos context (as in SequenceGenerator: tokens[:, 0] = eos)
            state = lm.init_incremental_state(None, B, beam)
            rows, _ = lm.decode_step(0, torch.full((N, 1), eos_lm, dtype=torch.int32, device=dev), state, None)
            lm_kw = dict(V_lm=n_lm, lm_blank=self.lm_blank, lm_weight=self.lm_weight)
            if T == 0:  # no frame to search: just the initial state
                _ops.ctc_beam_search(logits, V, lens, frames, beam, thr, 0, 0, ws, lm=rows, word_score=self.word_score,
                                     eos=self.eos, **lm_kw)
            for t in range(T):
                new_order, grown, fed = _ops.ctc_beam_search(logits, V, lens, frames, beam, thr, t, t + 1, ws, lm=rows,
                                                             word_score=self.word_score, eos=self.eos, want_order=True, **lm_kw)
                idx = new_order.long()
                old = {k: [s.index_select(0, idx) for s in state[k]] for k in ("h", "c")}
                new = {k: list(v) for k, v in old.items()}
                new_rows, _ = lm.decode_step(0, fed.view(N, 1), new, None)
                keep = grown.view(N, 1) == 0
                state = {k: [torch.where(keep, o, n) for o, n in zip(old[k], new[k])] for k in ("h", "c")}
                rows = torch.where(keep, rows.index_select(0, idx), new_rows)
            lm_kw["lm"] = rows
        res = _ops.ctc_beam_finalize(lens, T, V, beam, self.nbest, ws, eos=self.eos, pad=self.pad,
                                     want_frames=self.print_alignment, **lm_kw)
        return tuple(r.cpu() if r is not None else None for r in res)

    def generate(self, models, sample, **unused):
        if self.greedy:
            tokens, _, _ = self.decode(models, sample)
            return [[{"tokens": t[t != self.pad], "score": 0.0, "attention": None, "alignment": None, "positional_scores": None}]
                    for t in tokens]
        model = models[0]
        model.eval()
        with torch.no_grad():
            net = model(**sample["net_input"])
        tokens, lens, scores, frames = self.search(net["b200_out"], net["encoder_out"][0].size(-1), net["src_lengths"][0])
        out = []
        for b in range(tokens.size(0)):
            hyps = []
            for r in range(tokens.size(1)):
                s = float(scores[b, r])
                if s == -math.inf:
                    break
                n = int(lens[b, r])
                hyps.append({"tokens": tokens[b, r, :n].long(), "score": s, "attention": None,
                             "alignment": frames[b, r, :n].long() if frames is not None else None, "positional_scores": None})
            if not hyps:  # through a lexicon, a sentence whose last beam holds no whole-word hypothesis has none
                hyps.append({"tokens": torch.zeros(0, dtype=torch.long), "score": -math.inf, "attention": None,
                             "alignment": torch.zeros(0, dtype=torch.long) if frames is not None else None,
                             "positional_scores": None})
            out.append(hyps)
        return out
