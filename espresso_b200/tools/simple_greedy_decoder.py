"""Greedy decoder for encoder-decoder models, used by the reference for validation WER and teacher-free scoring
(espresso/tools/simple_greedy_decoder.py:18-166).

decode(models, sample) -> (tokens int64 [B, L] without the leading eos/bos, lprobs fp32 [B, U_target, V] or None, None):
the arg-max token of every step is fed back; a finished hypothesis keeps emitting eos; in validation mode the
decoding length is max(T', U_target) and the per-step log-probabilities of the first U_target steps are returned
(uniform where the hypothesis had already finished), exactly like the reference (:103-152).

One-token decoder steps run through the model's incremental-decoding protocol (decode_step: native embedding,
ancestor-indexed self-attention cache, un-replicated cross-attention, GEMMs) with beam 1; the arg-max is
esp_argmax_rows.  Only the tiny [B, V] log-softmax of validation mode uses torch."""
import math

import torch

from .. import ops as _ops


class SimpleGreedyDecoder:
    def __init__(self, models, dictionary, max_len_a=0, max_len_b=200, max_len=0, temperature=1.0, eos=None,
                 for_validation=True, **unused):
        self.models = models if isinstance(models, (list, tuple)) else [models]
        if len(self.models) != 1:
            raise NotImplementedError("ensembles are not on the native path yet")
        self.pad = dictionary.pad()
        self.eos = dictionary.eos() if eos is None else eos
        self.vocab_size = len(dictionary)
        self.max_len_a, self.max_len_b = max_len_a, max_len_b
        self.max_len = max_len or self.models[0].max_decoder_positions()
        assert temperature > 0, "--temperature must be greater than 0"
        self.temperature = temperature
        self.for_validation = for_validation

    @torch.no_grad()
    def decode(self, models, sample, bos_token=None, **unused):
        model = self.models[0]
        model.eval()
        net_input = sample["net_input"]
        src_tokens = net_input["src_tokens"]
        bsz, src_len = src_tokens.shape[:2]
        if src_tokens.dim() == 2 and src_tokens.is_floating_point():  # raw waveforms: T_src counts feature frames
            src_len = _ops.num_frames(src_len)
        dev = src_tokens.device
        enc = model.forward_encoder(net_input)
        target = sample.get("target")
        assert target is not None or not self.for_validation
        t_enc = enc["encoder_out"][0].size(0)
        if self.for_validation:
            max_len = max(t_enc, target.size(1))
        else:
            max_len = min(int(self.max_len_a * src_len + self.max_len_b), self.max_len - 1)
        if hasattr(model, "t_max_hint"):
            model.t_max_hint = max_len + 1
        state = model.init_incremental_state(enc, bsz, 1)
        V = self.vocab_size
        tokens = torch.full((bsz, max_len + 2), self.pad, dtype=torch.int32, device=dev)
        tokens[:, 0] = self.eos if bos_token is None else bos_token
        lprobs = None
        if self.for_validation:
            lprobs = torch.full((bsz, target.size(1), V), -math.log(V), dtype=torch.float32, device=dev)
        n_steps = max_len + 1
        for step in range(max_len + 1):  # one extra step for the eos marker
            is_eos = tokens[:, step] == self.eos
            if step > 0 and bool(is_eos.all()):
                n_steps = step
                break
            out, is_logits = model.decode_step(step, tokens, state, None)
            nxt = _ops.argmax_rows(out, V) if out.dtype == torch.bfloat16 else out[:, :V].argmax(-1)
            tokens[:, step + 1] = nxt.to(torch.int32)
            if step > 0:
                tokens[is_eos, step + 1] = self.eos  # finished hypotheses keep emitting eos
            if self.for_validation and step < target.size(1):
                x = out[:, :V].float()
                lp = torch.log_softmax(x / self.temperature, dim=-1) if is_logits else x
                if step > 0:
                    lp[is_eos, :] = -math.log(V)
                lprobs[:, step, :] = lp
        return tokens[:, 1: n_steps + 1].long(), lprobs, None

    def generate(self, models, sample, **kw):
        tokens, _, _ = self.decode(models, sample, **kw)
        out = []
        for t in tokens:
            t = t[t != self.pad]
            out.append([{"tokens": t, "score": 0.0, "attention": None, "alignment": None, "positional_scores": None}])
        return out
