"""Frame-synchronous greedy decoder for transducer models, the reference's validation / 1-best decoder
(espresso/tools/transducer_greedy_decoder.py:21-251, base class espresso/tools/transducer_base_decoder.py:17-190),
with optional shallow fusion of an LSTM language model (espresso_b200.models.LSTMLanguageModelEspresso; like the
reference, fusion needs an LM whose cached state can be rolled back per hypothesis).

Per encoder frame at most `max_num_expansions_per_step` non-blank tokens are emitted; a hypothesis that emits blank
moves to the next frame with its predictor state rolled back (`masked_copy_cached_state`), the last slot of a frame
records the blank score.  decode() returns (tokens int64 [B, T'*(E+1)] with blanks in the unused slots,
scores fp32 [B], None) like the reference's `_generate`.

The encoder runs once; its joint projection + LayerNorm is computed once for all frames.  Every expansion is: native
embedding lookup, two small GEMMs per LSTM layer (gates; the cell non-linearities on [B, 4H] are torch), projection +
LayerNorm, the joint add+ReLU kernel, the weight-normalised output GEMM, and a [B, V] log-softmax / arg-max."""
import torch

from .. import ops as _ops


class TransducerGreedyDecoder:
    def __init__(self, models, dictionary, max_len=0, max_num_expansions_per_step=2, temperature=1.0, eos=None, bos=None,
                 blank=None, model_predicts_eos=False, symbols_to_strip_from_output=None, lm_model=None, lm_weight=1.0,
                 print_alignment=False, **unused):
        self.model = (models if isinstance(models, (list, tuple)) else [models])[0]
        self.eos = dictionary.eos() if eos is None else eos
        self.bos = dictionary.eos() if bos is None else bos
        self.blank = dictionary.bos() if blank is None else blank  # the optional <s> symbol doubles as blank
        self.pad = dictionary.pad()
        self.model_predicts_eos = model_predicts_eos
        extra = set(symbols_to_strip_from_output or ())
        self.symbols_to_strip_from_output = extra | {self.eos, self.bos, self.blank}
        self.vocab_size = len(dictionary)
        self.max_len = max_len
        assert max_num_expansions_per_step > 0, "--max-num-expansions-per-step must be at least 1"
        self.max_num_expansions_per_step = max_num_expansions_per_step
        assert temperature > 0, "--temperature must be greater than 0"
        self.temperature = temperature
        self.print_alignment = print_alignment
        from ..models.ngram_lm import NgramLanguageModel

        if isinstance(lm_model, NgramLanguageModel):
            raise NotImplementedError("n-gram LMs are fused into CTC decoding only (CTCDecoder), not into transducer decoding")
        self.lm_model, self.lm_weight = lm_model, lm_weight
        self.no_blank_in_lm = False
        if lm_model is not None:
            dec = getattr(lm_model, "decoder", None)
            if dec is None or not hasattr(dec, "step"):
                raise NotImplementedError("transducer LM fusion needs an LSTM LM with a per-row cached state "
                                          "(masked_copy_cached_state in the reference)")
            n_lm = dec.embed_tokens.num_embeddings
            # an LM vocabulary one symbol short = the ASR vocabulary without blank (transducer_base_decoder.py:93-104)
            assert n_lm in (self.vocab_size, self.vocab_size - 1)
            self.no_blank_in_lm = n_lm == self.vocab_size - 1

    # ---- one predictor (LSTMCell stack) step from cached state --------------------------------------
    def _predictor_step(self, prev, hs, cs):
        m = self.model
        P = m.flat.param
        x = _ops.embed_fwd(prev.to(torch.int32), P("decoder.embed_tokens.weight"), None, 1, 1.0, self.pad)  # [B, E]
        nh, nc = [], []
        for i in range(len(m.decoder.layers)):
            p = "decoder.layers.%d." % i
            gates = _ops.linear(x, P(p + "weight_ih"), P(p + "bias_ih")).float() + \
                _ops.linear(hs[i], P(p + "weight_hh"), P(p + "bias_hh")).float()
            i_, f_, g_, o_ = gates.chunk(4, dim=1)
            c = torch.sigmoid(f_) * cs[i] + torch.sigmoid(i_) * torch.tanh(g_)
            h = (torch.sigmoid(o_) * torch.tanh(c)).to(torch.bfloat16)
            nh.append(h)
            nc.append(c)
            x = h
        return x, nh, nc

    @torch.no_grad()
    def decode(self, models, sample, bos_token=None, **unused):
        m = self.model
        m.eval()
        enc_out = m.forward_encoder(sample["net_input"])
        enc = enc_out["b200_out"]                                     # [B, T, d] bf16
        enc_lens = enc_out["src_lengths"][0].to(enc.device)
        B, T, d = enc.shape
        dev = enc.device
        t_max = int(enc_lens.max())
        max_len = min(t_max, self.max_len) if self.max_len > 0 else t_max
        E = self.max_num_expansions_per_step
        V = self.vocab_size
        pe_all = m.project(enc.reshape(B * T, d), "encoder")[0].view(B, T, -1)   # joint-space encoder frames, once
        W = m.fc_out_weight()[0]
        tokens = torch.full((B, max_len, E + 1), self.blank, dtype=torch.long, device=dev)
        scores = torch.zeros(B, max_len, E + 1, dtype=torch.float32, device=dev)
        prev = torch.full((B,), self.bos if bos_token is None else bos_token, dtype=torch.long, device=dev)
        hid = [l.weight_hh.shape[1] for l in m.decoder.layers]
        hs = [torch.zeros(B, h, dtype=torch.bfloat16, device=dev) for h in hid]
        cs = [torch.zeros(B, h, dtype=torch.float32, device=dev) for h in hid]
        lm = self.lm_model
        if lm is not None:
            lm.eval()
            lst = lm.init_incremental_state(None, B, 1)
            lhs, lcs = lst["h"], lst["c"]
            nonblank = torch.ones(V, dtype=torch.bool, device=dev)
            nonblank[self.blank] = False
        for t in range(max_len):
            blank_mask = t >= enc_lens
            k = 0
            pe_t = pe_all[:, t].contiguous().view(B, 1, -1)
            while k < E + 1 and not bool(blank_mask.all()):
                top, nh, nc = self._predictor_step(prev, hs, cs)
                pd = m.project(top, "decoder")[0]
                logits, _ = m.joint_logits(pe_t, pd.view(B, 1, -1), W)
                lp = torch.log_softmax(logits[:, :V].float() / self.temperature, dim=-1)
                if lm is not None:
                    # shallow fusion over the non-blank symbols, renormalised so that the transducer's blank / non-blank
                    # split is untouched (transducer_greedy_decoder.py:165-201)
                    lm_prev = torch.where(prev > self.blank, prev - 1, prev) if self.no_blank_in_lm else prev
                    ly, lnh, lnc, _ = lm.decoder.step(lm.decoder.embed_tokens(lm_prev), lhs, lcs, None)
                    lm_lp = torch.log_softmax(lm.decoder.output_layer(ly).float(), dim=-1)
                    if not self.no_blank_in_lm:
                        lm_lp = lm_lp[:, nonblank]
                    lp_nb = lp[:, nonblank]
                    fused = lp_nb + self.lm_weight * lm_lp
                    fused = fused + (lp_nb.exp().sum(1).log() - fused.exp().sum(1).log())[:, None]
                    lp[:, nonblank] = fused
                if self.model_predicts_eos:
                    # move the eos mass onto blank: mitigates early stops (transducer_greedy_decoder.py:203-208)
                    lp[:, self.blank] = torch.logaddexp(lp[:, self.blank], lp[:, self.eos])
                    lp[:, self.eos] = float("-inf")
                if k < E:
                    sc, tok = lp.max(-1)
                    scores[:, t, k] = torch.where(blank_mask, torch.zeros_like(sc), sc)
                    blank_mask = blank_mask | (tok == self.blank)
                    tokens[:, t, k] = torch.where(blank_mask, torch.full_like(tok, self.blank), tok)
                    prev = torch.where(blank_mask, prev, tok)
                else:  # the frame's last slot: score of the blank that ends it, if not emitted yet
                    scores[:, t, k] = torch.where(blank_mask, scores[:, t, k], lp[:, self.blank])
                    blank_mask = torch.ones_like(blank_mask)
                keep_old = blank_mask[:, None]  # masked_copy_cached_state: blank keeps the previous predictor state
                hs = [torch.where(keep_old, o, n) for o, n in zip(hs, nh)]
                cs = [torch.where(keep_old, o, n) for o, n in zip(cs, nc)]
                if lm is not None:
                    lhs = [torch.where(keep_old, o, n) for o, n in zip(lhs, lnh)]
                    lcs = [torch.where(keep_old, o, n) for o, n in zip(lcs, lnc)]
                k += 1
        alignments = tokens if self.print_alignment else None
        return tokens.view(B, -1), scores.view(B, -1).sum(-1), alignments

    def generate(self, models, sample, **kw):
        tokens, scores, alignments = self.decode(models, sample, **kw)
        strip = torch.tensor(sorted(self.symbols_to_strip_from_output), device=tokens.device)
        out = []
        for b in range(tokens.size(0)):
            t = tokens[b]
            t = t[~torch.isin(t, strip)]
            out.append([{"tokens": t, "score": scores[b], "attention": None,
                         "alignment": alignments[b] if alignments is not None else None, "positional_scores": None}])
        return out
