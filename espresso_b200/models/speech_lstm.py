"""`speech_lstm`: the attention-based LSTM encoder-decoder of BASELINE configs[0] (SURVEY.md §8a rows C3 / C4;
espresso/models/speech_lstm.py:170-1047, attention espresso/modules/speech_attention.py:38-95).

Scope note (SURVEY.md §2): the LSTM cells are not a north-star kernel and stay with cuDNN / ATen, here as in the
reference; this module is the host-level mirror that puts them behind the same model API as the other families --
reference state-dict keys, `build_model(cfg, task)`, `forward(src_tokens, src_lengths, prev_output_tokens)` returning
the teacher-forced logits -- so that the native pieces around them are the ones of this repository: the convolutional
front end's BatchNorm+ReLU kernels (ConvBNReLU), the fused label-smoothed cross-entropy criterion, the flat
parameter / gradient buffers with the single all-reduce and the fused Adam of the trainer.

  encoder : ConvBNReLU -> dropout -> per layer: pack -> (Bi)LSTM -> unpack -> dropout (not after the last) [+ residual]
  decoder : embedding -> per step: LSTMCell stack with input feeding; Bahdanau attention from the FIRST layer's hidden
            state; every deeper layer sees [hidden, context]; optional residuals; additional_fc; output projection"""
import math
from dataclasses import dataclass
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..flat import FlatParams
from ..registry import register_model
from .transformer.speech_transformer_encoder_model import ConvBNReLU, encoder_inputs


@dataclass
class SpeechLSTMModelConfig:
    dropout: float = 0.4
    encoder_conv_channels: Optional[str] = "[64, 64, 128, 128]"
    encoder_conv_kernel_sizes: Optional[str] = "[(3, 3), (3, 3), (3, 3), (3, 3)]"
    encoder_conv_strides: Optional[str] = "[(1, 1), (2, 2), (1, 1), (2, 2)]"
    encoder_rnn_hidden_size: int = 320
    encoder_rnn_layers: int = 3
    encoder_rnn_bidirectional: bool = True
    encoder_rnn_residual: bool = False
    decoder_embed_dim: int = 48
    decoder_hidden_size: int = 320
    decoder_layers: int = 3
    decoder_out_embed_dim: int = 960
    decoder_rnn_residual: bool = True
    attention_type: str = "bahdanau"
    attention_dim: int = 320
    share_decoder_input_output_embed: bool = False
    encoder_rnn_dropout_in: Optional[float] = None   # default: dropout
    encoder_rnn_dropout_out: Optional[float] = None
    decoder_dropout_in: Optional[float] = None
    decoder_dropout_out: Optional[float] = None
    max_source_positions: int = 10240
    max_target_positions: int = 1024
    # P_1, P_2, ...: probability of feeding the TRUTH token per epoch from start_scheduled_sampling_epoch on, the last value
    # for all later epochs (espresso/models/speech_lstm.py:150-165; asr_wsj / asr_swbd recipes)
    scheduled_sampling_probs: Tuple[float, ...] = (1.0,)
    start_scheduled_sampling_epoch: int = 1


class ScheduledSamplingRateScheduler:
    """espresso/tools/scheduled_sampling_rate_scheduler.py:10-45."""

    def __init__(self, scheduled_sampling_probs=(1.0,), start_scheduled_sampling_epoch=1):
        self.probs, self.start = list(scheduled_sampling_probs), start_scheduled_sampling_epoch

    def step(self, epoch):
        if (len(self.probs) > 1 or self.probs[0] < 1.0) and epoch >= self.start:
            return self.probs[min(epoch - self.start, len(self.probs) - 1)]
        return 1.0


def _uniform_(m, a=0.1):
    for n, p in m.named_parameters():
        if "weight" in n or "bias" in n:
            p.data.uniform_(-a, a)
    return m


class _BahdanauAttention(nn.Module):
    """score_t = v_n . tanh(W_q q + W_v value_t + b),  v_n = g * v / ||v||  (speech_attention.py:38-95)."""

    def __init__(self, query_dim, value_dim, embed_dim):
        super().__init__()
        self.query_proj = nn.Linear(query_dim, embed_dim, bias=False)
        self.value_proj = nn.Linear(value_dim, embed_dim, bias=False)
        self.v = nn.Parameter(torch.empty(embed_dim).uniform_(-0.1, 0.1))
        self.b = nn.Parameter(torch.zeros(embed_dim))
        self.g = nn.Parameter(torch.full((1,), math.sqrt(1.0 / embed_dim)))
        self.query_proj.weight.data.uniform_(-0.1, 0.1)
        self.value_proj.weight.data.uniform_(-0.1, 0.1)

    def keys(self, value):
        return self.value_proj(value)  # T x B x A, once per utterance batch

    def forward(self, query, value, key, key_padding_mask):
        vn = self.g * self.v / torch.norm(self.v)
        scores = (vn * torch.tanh(self.query_proj(query).unsqueeze(0) + key + self.b)).sum(dim=2)  # T x B
        if key_padding_mask is not None:
            scores = scores.float().masked_fill(key_padding_mask, float("-inf")).type_as(scores)
        w = F.softmax(scores, dim=0)
        return (w.unsqueeze(2) * value).sum(dim=0), w


class SpeechLSTMEncoder(nn.Module):
    def __init__(self, pre_encoder, input_size, hidden_size, num_layers, dropout_in, dropout_out, bidirectional, residual,
                 max_source_positions):
        super().__init__()
        self.pre_encoder = pre_encoder
        self.hidden_size, self.bidirectional, self.residual = hidden_size, bidirectional, residual
        self.dropout_in, self.dropout_out = dropout_in, dropout_out
        self.max_source_positions = max_source_positions
        self.output_units = hidden_size * (2 if bidirectional else 1)
        self.lstm = nn.ModuleList([
            _uniform_(nn.LSTM(input_size if i == 0 else self.output_units, hidden_size, bidirectional=bidirectional))
            for i in range(num_layers)])

    def output_lengths(self, in_lengths):
        return in_lengths if self.pre_encoder is None else self.pre_encoder.output_lengths(in_lengths)

    def max_positions(self):
        return self.max_source_positions

    def forward(self, src_tokens, src_lengths, src_lengths_cpu=None, **unused):
        if self.pre_encoder is not None:
            x, lens = self.pre_encoder(src_tokens, src_lengths)
            lens_cpu = self.pre_encoder.output_lengths(src_lengths_cpu if src_lengths_cpu is not None else src_lengths.cpu())
        else:
            x, lens = src_tokens, src_lengths
            lens_cpu = src_lengths_cpu if src_lengths_cpu is not None else src_lengths.cpu()
        T = x.size(1)
        pad = torch.arange(T, device=x.device)[None, :] >= lens.to(x.device)[:, None]  # B x T
        x = F.dropout(x, self.dropout_in, self.training).transpose(0, 1)  # T x B x C
        for i, rnn in enumerate(self.lstm):
            prev = x
            packed = nn.utils.rnn.pack_padded_sequence(x, lens_cpu.long(), enforce_sorted=True)
            out, _ = rnn(packed)
            x, _ = nn.utils.rnn.pad_packed_sequence(out, padding_value=0.0, total_length=T)
            if i < len(self.lstm) - 1:
                x = F.dropout(x, self.dropout_out, self.training)
            if self.residual and i > 0:
                x = x + prev
        return {"encoder_out": [x], "encoder_padding_mask": [pad.t()] if bool(pad.any()) else [], "encoder_embedding": [],
                "encoder_states": [], "src_tokens": [], "src_lengths": [lens]}


class SpeechLSTMDecoder(nn.Module):
    def __init__(self, dictionary, embed_dim, hidden_size, out_embed_dim, num_layers, dropout_in, dropout_out,
                 encoder_output_units, attn_dim, residual, share_input_output_embed, max_target_positions,
                 scheduled_sampling_rate_scheduler=None):
        super().__init__()
        self.scheduled_sampling_rate_scheduler = scheduled_sampling_rate_scheduler
        self.dictionary = dictionary
        V, pad = len(dictionary), dictionary.pad()
        self.hidden_size, self.encoder_output_units, self.residual = hidden_size, encoder_output_units, residual
        self.dropout_in, self.dropout_out = dropout_in, dropout_out
        self.share_input_output_embed = share_input_output_embed
        self.max_target_positions = max_target_positions
        self.embed_tokens = nn.Embedding(V, embed_dim, padding_idx=pad)
        nn.init.uniform_(self.embed_tokens.weight, -0.1, 0.1)
        nn.init.constant_(self.embed_tokens.weight[pad], 0)
        self.layers = nn.ModuleList([
            _uniform_(nn.LSTMCell(encoder_output_units + (embed_dim if i == 0 else hidden_size), hidden_size))
            for i in range(num_layers)])
        # encoder_output_units == 0: no attention / input feeding (the language-model case, espresso/models/lstm_lm.py)
        self.attention = _BahdanauAttention(hidden_size, encoder_output_units, attn_dim) if encoder_output_units > 0 else None
        if hidden_size + encoder_output_units != out_embed_dim:
            self.additional_fc = _uniform_(nn.Linear(hidden_size + encoder_output_units, out_embed_dim))
        if not share_input_output_embed:
            self.fc_out = _uniform_(nn.Linear(out_embed_dim, V))

    def max_positions(self):
        return self.max_target_positions

    def step(self, x_j, hs, cs, feed, enc=None, keys=None, mask=None):
        """One time step of the LSTMCell stack.  Returns (features of the top layer [B, H + C], hs, cs, feed)."""
        attend = self.attention is not None
        inp = torch.cat((x_j, feed), dim=1) if attend else x_j  # input feeding: previous step's context
        context = feed
        hs, cs = list(hs), list(cs)
        for i, cell in enumerate(self.layers):
            h, c = cell(inp, (hs[i], cs[i]))
            below = inp[:, : self.hidden_size] if (self.residual and i > 0) else None
            if attend and i == 0:  # attention is driven by the FIRST layer's hidden state
                context, _ = self.attention(h, enc, keys, mask)
            inp = F.dropout(torch.cat((h, context), dim=1) if attend else h, self.dropout_out, self.training)
            if below is not None:
                inp = torch.cat((inp[:, : self.hidden_size] + below, inp[:, self.hidden_size:]), dim=1) if attend else inp + below
            hs[i], cs[i] = h, c
        return inp, hs, cs, context

    def output_layer(self, y):
        if hasattr(self, "additional_fc"):
            y = F.dropout(self.additional_fc(y), self.dropout_out, self.training)
        if self.share_input_output_embed:
            return F.linear(y, self.embed_tokens.weight)
        return self.fc_out(y)

    def forward(self, prev_output_tokens, encoder_out=None, epoch=1):
        """Teacher forcing, or -- in training, when the scheduler's probability of feeding the truth is < 1 -- scheduled
        sampling exactly as espresso/models/speech_lstm.py:735-764: at every step > 0 a per-sentence coin decides between
        the truth token and the arg-max of the previous step's output."""
        sampling_prob = 1.0
        if self.training and self.scheduled_sampling_rate_scheduler is not None:
            sampling_prob = self.scheduled_sampling_rate_scheduler.step(epoch)
        enc = mask = keys = None
        if self.attention is not None:
            enc = encoder_out["encoder_out"][0]                                     # T x B x C
            mask = encoder_out["encoder_padding_mask"][0] if encoder_out["encoder_padding_mask"] else None
            keys = self.attention.keys(enc)
        B, U = prev_output_tokens.shape
        x = F.dropout(self.embed_tokens(prev_output_tokens), self.dropout_in, self.training).transpose(0, 1)
        hs = [x.new_zeros(B, self.hidden_size) for _ in self.layers]
        cs = [x.new_zeros(B, self.hidden_size) for _ in self.layers]
        feed = x.new_zeros(B, self.encoder_output_units) if self.attention is not None else None
        outs = []
        if sampling_prob >= 1.0:
            for j in range(U):
                y, hs, cs, feed = self.step(x[j], hs, cs, feed, enc, keys, mask)
                outs.append(y)
            return self.output_layer(torch.stack(outs, dim=1))                      # B x U x V
        logits, pred = [], None
        for j in range(U):
            tok = prev_output_tokens[:, j]
            if j > 0:
                use_truth = torch.rand(B, device=tok.device).lt(sampling_prob)
                tok = torch.where(use_truth, tok, pred)
            x_j = F.dropout(self.embed_tokens(tok), self.dropout_in, self.training)
            y, hs, cs, feed = self.step(x_j, hs, cs, feed, enc, keys, mask)
            lj = self.output_layer(y)                                               # B x V
            logits.append(lj)
            pred = lj.argmax(-1)
        return torch.stack(logits, dim=1)


@register_model("speech_lstm", dataclass=SpeechLSTMModelConfig)
class SpeechLSTMModel(nn.Module):
    def __init__(self, encoder, decoder):
        super().__init__()
        self.encoder, self.decoder = encoder, decoder
        self.num_updates = 0
        self._flat = None

    @classmethod
    def build_model(cls, cfg, task):
        if str(cfg.attention_type).lower() != "bahdanau":
            raise NotImplementedError("speech_lstm on the native path: Bahdanau attention (the recipes' setting)")
        if cfg.share_decoder_input_output_embed and cfg.decoder_embed_dim != cfg.decoder_out_embed_dim:
            raise ValueError("--share-decoder-input-output-embed requires --decoder-embed-dim to match --decoder-out-embed-dim")
        conv, size = ConvBNReLU.from_config(cfg.encoder_conv_channels, cfg.encoder_conv_kernel_sizes, cfg.encoder_conv_strides,
                                            task.feat_dim, task.feat_in_channels)
        d = lambda v: cfg.dropout if v is None else v  # noqa: E731
        enc = SpeechLSTMEncoder(conv, size, cfg.encoder_rnn_hidden_size, cfg.encoder_rnn_layers, d(cfg.encoder_rnn_dropout_in),
                                d(cfg.encoder_rnn_dropout_out), cfg.encoder_rnn_bidirectional, cfg.encoder_rnn_residual,
                                cfg.max_source_positions)
        dec = SpeechLSTMDecoder(task.target_dictionary, cfg.decoder_embed_dim, cfg.decoder_hidden_size, cfg.decoder_out_embed_dim,
                                cfg.decoder_layers, d(cfg.decoder_dropout_in), d(cfg.decoder_dropout_out), enc.output_units,
                                cfg.attention_dim, cfg.decoder_rnn_residual, cfg.share_decoder_input_output_embed,
                                cfg.max_target_positions,
                                scheduled_sampling_rate_scheduler=ScheduledSamplingRateScheduler(
                                    getattr(cfg, "scheduled_sampling_probs", (1.0,)),
                                    getattr(cfg, "start_scheduled_sampling_epoch", 1)))
        return cls(enc, dec)

    # ---- native wiring: flat buffers (one all-reduce, fused Adam), native BatchNorm in the conv front ----------------
    def finalize_(self, device):
        self.to(device)
        pe = self.encoder.pre_encoder
        self._flat = FlatParams(self, device=device,
                                channels_last=pe.channels_last_weights("encoder.pre_encoder.") if pe is not None else ())
        if pe is not None:
            pe.use_flat_(self._flat, "encoder.pre_encoder.")
        # (no rnn.flatten_parameters(): cuDNN would move the weights out of the flat buffer the optimizer updates)
        return self

    @property
    def flat(self):
        return self._flat

    def sync_torch_grads_(self):
        """Fold the bf16 .grad of the torch-executed parameters (convolutions, LSTMs, attention, projections) into the
        flat fp32 gradient buffer; BatchNorm parameters were accumulated there by the native kernels already."""
        self._flat.fold_torch_grads_(self)

    def set_num_updates(self, n):
        self.num_updates = n

    def max_positions(self):
        return (self.encoder.max_positions(), self.decoder.max_positions())

    def max_decoder_positions(self):
        return self.decoder.max_positions()

    def output_lengths(self, in_lengths):
        return self.encoder.output_lengths(in_lengths)

    def forward(self, src_tokens, src_lengths, prev_output_tokens, epoch=1, src_lengths_cpu=None, freq_masks=None,
                time_masks=None, time_warp=None, **unused):
        src_tokens, src_lengths, src_lengths_cpu = encoder_inputs(self, src_tokens, src_lengths, src_lengths_cpu, freq_masks,
                                                                  time_masks, time_warp)
        enc = self.encoder(src_tokens.to(self.decoder.embed_tokens.weight.dtype), src_lengths, src_lengths_cpu=src_lengths_cpu)
        logits = self.decoder(prev_output_tokens, enc, epoch=epoch)                  # B x U x V
        V = logits.size(-1)
        ldV = (V + 7) // 8 * 8
        padded = F.pad(logits, (0, ldV - V)) if ldV != V else logits
        return padded[..., :V], {"attn": None, "b200_out": padded.contiguous()}

    def get_normalized_probs(self, net_output, log_probs, sample=None):
        x = net_output[0].float()
        return F.log_softmax(x, dim=-1) if log_probs else F.softmax(x, dim=-1)

    # ---- generator protocol (espresso_b200/sequence_generator.py): incremental decoding with cached (h, c, context) ---
    def forward_encoder(self, net_input):
        src = net_input["src_tokens"].to(self.decoder.embed_tokens.weight.dtype)
        return self.encoder(src, net_input["src_lengths"], src_lengths_cpu=net_input.get("src_lengths_cpu"))

    def init_incremental_state(self, encoder_out, bsz, beam):
        """Encoder outputs (and the attention keys, computed once) are replicated per hypothesis; a search step only
        permutes hypotheses inside a sentence, so they never need reordering (reorder_encoder_out in the reference)."""
        dec = self.decoder
        enc = encoder_out["encoder_out"][0].repeat_interleave(beam, dim=1)            # T x N x C
        mask = encoder_out["encoder_padding_mask"][0].repeat_interleave(beam, dim=1) if encoder_out["encoder_padding_mask"] else None
        N = bsz * beam
        z = lambda w: [enc.new_zeros(N, w) for _ in dec.layers]  # noqa: E731
        return {"enc": enc, "mask": mask, "keys": dec.attention.keys(enc), "h": z(dec.hidden_size), "c": z(dec.hidden_size),
                "feed": enc.new_zeros(N, dec.encoder_output_units)}

    @torch.no_grad()
    def decode_step(self, step, tokens, state, new_order):
        dec = self.decoder
        if new_order is not None:  # reorder_incremental_state (speech_lstm.py:974-1000)
            idx = new_order.long()
            state["h"] = [h.index_select(0, idx) for h in state["h"]]
            state["c"] = [c.index_select(0, idx) for c in state["c"]]
            state["feed"] = state["feed"].index_select(0, idx)
        x = dec.embed_tokens(tokens[:, step].long())
        y, state["h"], state["c"], state["feed"] = dec.step(x, state["h"], state["c"], state["feed"], state["enc"], state["keys"],
                                                             state["mask"])
        logits = dec.output_layer(y)
        V = logits.size(-1)
        ldV = (V + 7) // 8 * 8
        if logits.dtype == torch.bfloat16 and ldV != V:
            logits = F.pad(logits, (0, ldV - V))
        return logits.contiguous(), True
