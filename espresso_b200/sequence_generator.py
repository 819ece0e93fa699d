"""Batched beam search with LM shallow fusion, H100-native mirror of `SequenceGenerator`
(fairseq/sequence_generator.py:27-621 with the Espresso patches: lm_model / lm_weight :385-393, eos_factor
:404-410) and `BeamSearch.step` (fairseq/search.py:103-144).

generate(models, sample) -> List[bsz] of List[<= beam] of {"tokens" (ends with eos), "score", "attention",
"alignment", "positional_scores"}, sorted by score -- the reference's contract (:744-752).  "attention" is None unless the
generator was built with print_alignment and every model records encoder attention (decode_attention below); it is then
fp32 [T', len(tokens)] on the host, column t = the last decoder layer's head-averaged encoder attention at step t of the
hypothesis's ancestor (:429-435,603-605,690,739-748; ensembles: the mean over models, :889-900).  "alignment" stays None.

The per-step tensor work is three native kernels (esp_beam_merge, esp_beam_topk, esp_beam_bookkeep) plus
esp_gather_rows for the incremental state; hypothesis bookkeeping and finalisation live in device buffers, and the
only host<->device traffic per step is one 4-byte "how many sentences are unfinished" read.  Finished sentences are
kept in the batch (static shapes) instead of being compacted away (:507-541): results are identical.
fairseq's search options change only the step between merge and bookkeeping (csrc/beam_options.cu): prefix_tokens
(:414-424,623-657), no_repeat_ngram_size (:448-449), diverse_beam_groups / diverse_beam_strength (DiverseBeamSearch) and
diversity_rate (DiverseSiblingsSearch), sampling / sampling_topk / sampling_topp (Sampling, drawn with a seed that advances
per generate() call).

Model protocol (implemented by espresso_b200 models and by test doubles):
    enc = model.forward_encoder(net_input)                       # any object
    model.max_decoder_positions() -> int
    state = model.init_incremental_state(enc, bsz, beam)          # encoder state replicated per beam if needed
    values, is_logits = model.decode_step(step, tokens, state, new_order)
        tokens: int32 [bsz*beam, max_len+2] device buffer (columns 0..step are valid);
        new_order: int32 [bsz*beam] source row of each hypothesis since the previous step (None at step 0);
        values: [bsz*beam, >= V] bf16/fp32 logits (is_logits) or fp32 log-probabilities.
Optional, for print_alignment:
    state = model.init_incremental_state(enc, bsz, beam, attention=True)
    attn, anc = model.decode_attention(state)   # after decode_step: the row of hypothesis n at step t is attn[t][anc[t][n]]
"""
import math

import torch

from . import ops as _ops


class _SearchState:
    pass


class SequenceGenerator:
    def __init__(self, models, tgt_dict, beam_size=1, max_len_a=0, max_len_b=200, max_len=0, min_len=1,
                 normalize_scores=True, len_penalty=1.0, unk_penalty=0.0, temperature=1.0, lm_model=None, lm_weight=1.0,
                 eos_factor=None, eos=None, use_cuda_graphs=True, print_alignment=None, no_repeat_ngram_size=0,
                 search_strategy=None, sampling=False, sampling_topk=-1, sampling_topp=-1.0, diverse_beam_groups=-1,
                 diverse_beam_strength=0.5, diversity_rate=-1.0, sampling_seed=1, **unused):
        self.models = models if isinstance(models, (list, tuple)) else [models]
        assert len(self.models) >= 1
        self.tgt_dict = tgt_dict
        self.pad, self.unk = tgt_dict.pad(), tgt_dict.unk()
        self.eos = tgt_dict.eos() if eos is None else eos
        self.vocab_size = len(tgt_dict)
        self.beam_size = min(beam_size, self.vocab_size - 1)
        self.max_len_a, self.max_len_b, self.min_len = max_len_a, max_len_b, min_len
        self.max_len = max_len or self.models[0].max_decoder_positions()
        self.normalize_scores, self.len_penalty, self.unk_penalty = normalize_scores, len_penalty, unk_penalty
        self.temperature = temperature
        assert temperature > 0, "--temperature must be greater than 0"
        from .models.ngram_lm import NgramLanguageModel

        if isinstance(lm_model, NgramLanguageModel):
            raise NotImplementedError("n-gram LMs are fused into CTC decoding only (CTCDecoder), not into SequenceGenerator")
        self.lm_model, self.lm_weight = lm_model, lm_weight
        self.eos_factor = eos_factor
        assert eos_factor is None or eos_factor >= 1.0, "--eos-factor must be >= 1.0 if set"
        # One search step (decoder + LM step, merge, top-k, bookkeeping: ~140 kernel launches) is host-bound when launched
        # from Python.  With use_cuda_graphs every step index gets its own CUDA graph over PERSISTENT search / decoder state
        # (first batch of a shape: eager, second: capture, then replay); the per-step "all sentences finished?" read stays
        # outside the graphs.  Single-model search only (ensembles run eagerly).
        self.use_cuda_graphs = use_cuda_graphs
        self._graph_cache = {}
        # any truthy value (the reference's "hard" / "soft"): record each hypothesis's encoder attention
        self.print_alignment = bool(print_alignment)
        # search options (fairseq/search.py); a fairseq search object may be passed instead of the keywords
        if search_strategy is not None:
            sampling, sampling_topk, sampling_topp, diverse_beam_groups, diverse_beam_strength, diversity_rate = \
                _search_keywords(search_strategy)
        if sum(int(c) for c in (bool(sampling), diverse_beam_groups > 0, diversity_rate > 0)) > 1:
            raise ValueError("Provided Search parameters are mutually exclusive.")
        assert sampling_topk < 0 or sampling, "--sampling-topk requires --sampling"
        assert sampling_topp < 0 or sampling, "--sampling-topp requires --sampling"
        self.sampling, self.sampling_topk, self.sampling_topp = bool(sampling), int(sampling_topk), float(sampling_topp)
        # the sampling seed: generate() call c draws with seed sampling_seed + c, read by the kernel from device memory
        self._next_seed = int(sampling_seed)
        if diverse_beam_groups > 0 and self.beam_size % diverse_beam_groups != 0:
            raise ValueError("DiverseBeamSearch requires --beam to be divisible by the number of groups")
        self.diverse_beam_groups, self.diverse_beam_strength = int(diverse_beam_groups), float(diverse_beam_strength)
        self.diversity_rate = float(diversity_rate) if diverse_beam_groups <= 0 and not sampling else -1.0
        if sampling:
            self.diverse_beam_groups = -1
        self.no_repeat_ngram_size = int(no_repeat_ngram_size or 0)

    @torch.no_grad()
    def generate(self, models, sample, **kwargs):
        return self._generate(sample, **kwargs)

    def forward(self, sample, **kwargs):
        return self._generate(sample, **kwargs)

    @torch.no_grad()
    def _generate(self, sample, prefix_tokens=None, bos_token=None, **unused):
        model = self.models[0]
        net_input = sample["net_input"]
        src_tokens = net_input["src_tokens"]
        dev = src_tokens.device
        bsz, src_len = src_tokens.shape[:2]
        if src_tokens.dim() == 2 and src_tokens.is_floating_point():
            # raw waveform batch [B, samples] (on-device front end): the reference's T_src is the padded number of
            # feature FRAMES (src_tokens.size(1) of [B, T, F], sequence_generator.py:270,285-288)
            src_len = _ops.num_frames(src_len)
        beam, V = self.beam_size, self.vocab_size
        max_len = min(int(self.max_len_a * src_len + self.max_len_b), self.max_len - 1)  # :285-288
        assert self.min_len <= max_len, "min_len cannot be larger than max_len, please adjust these!"
        N, L = bsz * beam, max_len + 2
        P = 0 if prefix_tokens is None else int(prefix_tokens.shape[1])
        if P > 0 and bool(((prefix_tokens < 0) | (prefix_tokens >= V)).any()):
            raise ValueError("prefix_tokens must lie in [0, %d)" % V)

        for m_ in tuple(self.models) + (self.lm_model,):
            if m_ is not None and hasattr(m_, "t_max_hint"):
                m_.t_max_hint = max_len + 1
        graphs_on = (self.use_cuda_graphs and dev.type == "cuda" and len(self.models) == 1
                     and hasattr(model, "advance_state_without_compute")
                     and (self.lm_model is None or hasattr(self.lm_model, "advance_state_without_compute")))
        enc = model.forward_encoder(net_input)
        cache = None
        if graphs_on:
            enc_T = enc["b200_out"].shape[1] if isinstance(enc, dict) and "b200_out" in enc else -1
            has_pad = isinstance(enc, dict) and len(enc.get("encoder_padding_mask", [])) > 0
            key = (bsz, beam, max_len, enc_T, has_pad, bos_token, str(dev), self.print_alignment, P)
            cache = self._graph_cache.get(key)
            if cache is None:
                if len(self._graph_cache) >= 4:  # bounded: search shapes come in a handful of buckets
                    self._graph_cache.pop(next(iter(self._graph_cache)))
                cache = self._graph_cache[key] = {"calls": 0, "graphs": {}, "pool": None, "state": None, "lm_state": None,
                                                  "search": None}
        # an ensemble = one encoder pass and one incremental state per model; their step log-probs are averaged in the
        # probability domain (EnsembleModel.forward_decoder, fairseq/sequence_generator.py:836-901)
        want_attn = self.print_alignment and all(hasattr(m_, "decode_attention") for m_ in self.models)
        akw = {"attention": True} if want_attn else {}
        if graphs_on:
            states = [model.init_incremental_state(enc, bsz, beam, reuse=cache["state"], **akw)]
            cache["state"] = states[0]
        else:
            states = [model.init_incremental_state(enc, bsz, beam, **akw)]
            for m_ in self.models[1:]:
                states.append(m_.init_incremental_state(m_.forward_encoder(net_input), bsz, beam, **akw))
        state = states[0]
        want_attn = want_attn and all(m_.decode_attention(s_) is not None for m_, s_ in zip(self.models, states))
        lm_state = None
        if self.lm_model is not None:
            if graphs_on:
                lm_state = cache["lm_state"] = self.lm_model.init_incremental_state(None, bsz, beam, reuse=cache["lm_state"])
            else:
                lm_state = self.lm_model.init_incremental_state(None, bsz, beam)
        for s_ in states + [lm_state]:  # models may size their caches from this
            if isinstance(s_, dict):
                s_["max_len"] = max_len

        st = cache["search"] if graphs_on else None
        if st is None:
            st = _SearchState()
            st.buf_tokens = [torch.empty((N, L), dtype=torch.int32, device=dev) for _ in range(2)]
            st.buf_scores = [torch.empty(N, L - 1, dtype=torch.float32, device=dev) for _ in range(2)]
            st.ignore = torch.empty(N, dtype=torch.uint8, device=dev)
            st.finished = torch.empty(bsz, dtype=torch.uint8, device=dev)
            st.nfin = torch.empty(bsz, dtype=torch.int32, device=dev)
            st.fin_tokens = torch.empty((bsz, beam, L - 1), dtype=torch.int32, device=dev)
            st.fin_len = torch.empty(bsz, beam, dtype=torch.int32, device=dev)
            st.fin_score = torch.empty(bsz, beam, dtype=torch.float32, device=dev)
            st.fin_pos = torch.empty(bsz, beam, L - 1, dtype=torch.float32, device=dev)
            st.new_order = torch.empty(N, dtype=torch.int32, device=dev)
            st.n_unfinished = torch.empty((1,), dtype=torch.int32, device=dev)
            st.cand = torch.empty(N, V, dtype=torch.float32, device=dev)
            st.prev = torch.empty(N, dtype=torch.float32, device=dev)
            st.arange = torch.arange(N, dtype=torch.int32, device=dev)
            if P > 0:
                st.prefix = torch.empty(bsz, P, dtype=torch.int32, device=dev)
            if self.sampling:
                st.seed = torch.empty(1, dtype=torch.int64, device=dev)
            if want_attn:  # [bsz, beam, L - 1, T']: row t of a finalised hypothesis = its attention at step t
                Tk = model.decode_attention(state)[0].shape[2]
                st.fin_attn = torch.empty(bsz, beam, L - 1, Tk, dtype=torch.float32, device=dev)
            if graphs_on:
                cache["search"] = st
        # (re-)initialise in place: the same buffers, in the same ping-pong roles, for every batch of this shape
        st.tokens, st.tokens_alt = st.buf_tokens
        st.scores, st.scores_alt = st.buf_scores
        st.tokens.fill_(self.pad)
        st.tokens[:, 0] = self.eos if bos_token is None else bos_token
        st.scores.zero_()
        st.scores_alt.zero_()
        st.ignore.zero_()
        st.finished.zero_()
        st.nfin.zero_()
        st.fin_tokens.fill_(self.pad)
        st.fin_len.zero_()
        st.fin_score.zero_()
        st.fin_pos.zero_()
        st.new_order.copy_(st.arange)
        st.n_unfinished.fill_(bsz)
        if P > 0:
            st.prefix.copy_(prefix_tokens)
        if self.sampling:
            st.seed.fill_(self._next_seed)
            self._next_seed += 1
        cand, prev = st.cand, st.prev
        groups = self.diverse_beam_groups

        def device_step(step):
            """All device work of search step `step` (this is what a step graph records)."""
            new_order = st.new_order if step > 0 else None
            values, is_logits = model.decode_step(step, st.tokens, state, new_order)
            if len(self.models) > 1:
                lps = []
                for m_, s_ in zip(self.models, states):
                    v_, il_ = (values, is_logits) if m_ is model else m_.decode_step(step, st.tokens, s_, new_order)
                    v_ = v_[:, :V].float()
                    lps.append(torch.log_softmax(v_ / self.temperature, dim=-1) if il_ else v_)
                values = torch.logsumexp(torch.stack(lps, dim=0), dim=0) - math.log(len(self.models))
                is_logits = False  # temperature already applied per model (sequence_generator.py:866-870)
            lm_vals, lm_logits = (None, True)
            if self.lm_model is not None:
                lm_vals, lm_logits = self.lm_model.decode_step(step, st.tokens, lm_state, new_order)
            # the merge adds the cumulative scores, except for the diverse groups, whose penalty comes first, and for
            # sampling, which draws from the step's own probabilities
            merge_prev = step > 0 and groups <= 0 and not self.sampling
            if merge_prev:
                prev.copy_(st.scores[:, step - 1])
            forced = step < P and step < max_len  # prefix tokens; the min-length eos ban is off there (:414-424)
            _ops.beam_merge(values, V, is_logits, cand, prev_scores=prev if merge_prev else None,
                            temperature=self.temperature if (is_logits or len(self.models) == 1) else 1.0,
                            lm=lm_vals, lm_is_logits=lm_logits, lm_weight=self.lm_weight, pad=self.pad, unk=self.unk,
                            unk_penalty=self.unk_penalty, eos=self.eos, force_eos=step >= max_len,
                            eos_factor=self.eos_factor, ban_eos=step < self.min_len and not forced)
            if forced:
                _ops.beam_prefix(st.prefix, step, beam, self.pad, self.eos, cand, V, st)
            if self.no_repeat_ngram_size > 0:
                _ops.beam_block_ngrams(st.tokens, step, self.no_repeat_ngram_size, cand, V)
            n_cand = V if step == 0 else beam * V  # step 0: all beams are identical, use the first (search.py:119-122)
            if (groups > 0 or self.sampling) and step > 0:  # after the prefix step, which may copy beam 0's scores
                prev.copy_(st.scores[:, step - 1])
            if self.sampling:
                K = beam  # one draw per hypothesis (search.py:700-715)
                cs, ct, cb = _ops.beam_sample(cand, prev if step > 0 else None, bsz, beam, V, self.sampling_topk,
                                              self.sampling_topp, st.seed, step)
            elif groups > 0:
                Kg = min(2 * (beam // groups), n_cand // groups - 1 if step > 0 else V - 1)
                K = Kg * groups
                cs, ct, cb = _ops.beam_diverse_groups(cand, prev if step > 0 else None, bsz, beam, V, groups, Kg,
                                                      self.diverse_beam_strength)
            elif self.diversity_rate > -1 and step > 0:
                K = min(2 * beam, n_cand - 1)
                cs, ct, cb = _ops.beam_sibling_topk(cand, bsz, beam, V, K, self.diversity_rate)
            else:
                K = min(2 * beam, n_cand - 1)
                cs, ct, cb = _ops.beam_topk(cand, bsz, beam * V, n_cand, K, V)
            if not want_attn:
                _ops.beam_bookkeep(step, max_len, bsz, beam, K, self.eos, self.pad, self.normalize_scores, self.len_penalty,
                                   cs, ct, cb, st)
                return
            att, anc = model.decode_attention(state)
            if len(self.models) > 1:  # the members' rows are averaged before they enter the history (:889-900)
                for m_, s_ in zip(self.models[1:], states[1:]):
                    att[step].add_(m_.decode_attention(s_)[0][step])
                att[step].div_(len(self.models))
            _ops.beam_bookkeep_attn(step, max_len, bsz, beam, K, self.eos, self.pad, self.normalize_scores, self.len_penalty,
                                    cs, ct, cb, st, att, anc)

        def host_swaps():
            """What device_step changes on the host side (ping-pong roles); replays must repeat it."""
            st.tokens, st.tokens_alt = st.tokens_alt, st.tokens
            st.scores, st.scores_alt = st.scores_alt, st.scores
            model.advance_state_without_compute(state)
            if self.lm_model is not None:
                self.lm_model.advance_state_without_compute(lm_state)

        # "all sentences finished?" is read one step LATE through pinned memory: the host never waits for the step it has
        # just queued (finished sentences are inert, so at most one surplus step runs after the last hypothesis ended)
        lagged = dev.type == "cuda"
        if lagged:
            if not hasattr(self, "_nu_host"):
                self._nu_host = [torch.zeros(1, dtype=torch.int32).pin_memory() for _ in range(2)]
                self._nu_ev = [torch.cuda.Event() for _ in range(2)]
        for step in range(max_len + 1):  # one extra step for the eos marker
            graph = cache["graphs"].get(step) if graphs_on else None
            if graph is not None:
                graph.replay()
                host_swaps()
            elif graphs_on and cache["calls"] >= 1:
                # second batch of this shape: record the step (recording executes nothing), then run it by replaying
                graph = torch.cuda.CUDAGraph()
                torch.cuda.synchronize()
                with torch.cuda.graph(graph, pool=cache["pool"]):
                    device_step(step)
                if cache["pool"] is None:
                    cache["pool"] = graph.pool()
                cache["graphs"][step] = graph
                graph.replay()
            else:
                device_step(step)
            if lagged:
                k = step & 1
                self._nu_host[k].copy_(st.n_unfinished, non_blocking=True)
                self._nu_ev[k].record()
                if step > 0:
                    self._nu_ev[1 - k].synchronize()
                    if int(self._nu_host[1 - k][0]) == 0:
                        break
            elif int(st.n_unfinished.item()) == 0:
                break
        if graphs_on:
            cache["calls"] += 1

        # ---- collect (:611-620): sort each sentence's hypotheses by score, descending
        nfin = st.nfin.cpu().tolist()
        fl, fs = st.fin_len.cpu(), st.fin_score.cpu()
        ft, fp = st.fin_tokens.cpu(), st.fin_pos.cpu()
        fa = st.fin_attn[:, :, :max(1, int(fl.max()))].cpu() if want_attn else None
        finalized = []
        for s in range(bsz):
            hyps = []
            for k in range(nfin[s]):
                n = int(fl[s, k])
                hyps.append({"tokens": ft[s, k, :n].long(), "score": fs[s, k].clone(),
                             "attention": fa[s, k, :n].T.contiguous() if want_attn else None, "alignment": None,
                             "positional_scores": fp[s, k, :n].clone()})
            order = sorted(range(len(hyps)), key=lambda i: -float(hyps[i]["score"]))
            finalized.append([hyps[i] for i in order])
        return finalized


def _search_keywords(search):
    """A fairseq search object (fairseq/search.py) -> (sampling, sampling_topk, sampling_topp, diverse_beam_groups,
    diverse_beam_strength, diversity_rate)."""
    name = type(search).__name__
    if name == "BeamSearch":
        return False, -1, -1.0, -1, 0.5, -1.0
    if name == "Sampling":
        return True, search.sampling_topk, search.sampling_topp, -1, 0.5, -1.0
    if name == "DiverseBeamSearch":  # stores -strength (search.py:563)
        return False, -1, -1.0, search.num_groups, -search.diversity_strength, -1.0
    if name == "DiverseSiblingsSearch":
        return False, -1, -1.0, -1, 0.5, search.diversity_rate
    raise NotImplementedError("search strategy %s is not supported by the native SequenceGenerator" % name)


class TableDecoderModel:
    """Decoder double driven by per-step probability tables (the reference's TestIncrementalDecoder,
    tests/utils.py:546-603): used to run the reference's known-answer beam-search tests against this generator."""

    def __init__(self, beam_probs, vocab_size, eos, max_positions=100):
        self.beam_probs, self.V, self.eos, self.max_pos = beam_probs, vocab_size, eos, max_positions

    def max_decoder_positions(self):
        return self.max_pos

    def forward_encoder(self, net_input):
        return None

    def init_incremental_state(self, enc, bsz, beam):
        return {"order": None}

    def decode_step(self, step, tokens, state, new_order):
        N = tokens.shape[0]
        probs = torch.zeros(N, self.V, dtype=torch.float32)
        if step < len(self.beam_probs):
            t = self.beam_probs[step]
            probs[:, self.eos:] = t if t.shape[0] == N else t[: N]
        else:
            probs[:, self.eos] = 1.0
        return probs.log().to(tokens.device), False
