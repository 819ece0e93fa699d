"""`speech_transformer_base` (Transformer/Conformer encoder + Transformer decoder), H100-native.

Mirrors espresso/models/transformer/speech_transformer_base.py:28-260 (SpeechTransformerModelBase:
build_model / forward(src_tokens, src_lengths, prev_output_tokens, epoch=) -> (logits [B,U,V], extra) /
get_normalized_probs / max_positions) and espresso/models/transformer/speech_transformer_decoder.py:43-281.
State-dict keys equal the reference's.  Training (teacher forcing) runs in EncoderEngine + DecoderEngine.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from ...flat import FlatParams
from ...modules.decoder_engine import DecoderEngine, IncrementalDecoder
from ...registry import register_model
from .speech_transformer_config import DEFAULT_MAX_SOURCE_POSITIONS, SpeechTransformerConfig
from .speech_transformer_encoder_model import (ConvBNReLU, SpeechTransformerEncoderForPrediction, _Affine, _Linear,
                                               _PosEmbStub, encoder_inputs)

DEFAULT_MAX_TARGET_POSITIONS = 1024


class _DecAttn(nn.Module):
    def __init__(self, d, self_attention):
        super().__init__()
        g = 1 / math.sqrt(2) if self_attention else 1.0  # qkv_same_dim init (multihead_attention.py:190-200)
        self.k_proj = _Linear(d, d, xavier=g)
        self.v_proj = _Linear(d, d, xavier=g)
        self.q_proj = _Linear(d, d, xavier=g)
        self.out_proj = _Linear(d, d, xavier=1.0)


class _DecoderLayer(nn.Module):
    def __init__(self, d, ffn):
        super().__init__()
        self.self_attn = _DecAttn(d, True)
        self.self_attn_layer_norm = _Affine(d)
        self.encoder_attn = _DecAttn(d, True)
        self.encoder_attn_layer_norm = _Affine(d)
        self.fc1 = _Linear(d, ffn, xavier=1.0)
        self.fc2 = _Linear(ffn, d, xavier=1.0)
        self.final_layer_norm = _Affine(d)


class _DecoderFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, enc, engine, tokens, enc_lens, tgt_lens):
        ctx.engine = engine
        return engine.forward(tokens, enc, enc_lens, tgt_lens)

    @staticmethod
    def backward(ctx, dlogits):
        return ctx.engine.backward(dlogits.contiguous()), None, None, None, None


class SpeechTransformerDecoderBase(nn.Module):
    def __init__(self, cfg: SpeechTransformerConfig, dictionary, embed_tokens):
        super().__init__()
        dc = cfg.decoder
        if dc.relative_positional_embeddings or dc.learned_pos or not dc.normalize_before:
            raise NotImplementedError("native decoder: pre-LN layers with sinusoidal absolute positions (the recipes' setting)")
        if dc.relaxed_attention_weight > 0 and any(p_ < 1.0 for p_ in getattr(cfg, "scheduled_sampling_probs", (1.0,))):
            # the reference relaxes the encoder attention of the sampled pass as well, which the native one does not model
            raise NotImplementedError("native decoder: relaxed encoder attention together with scheduled sampling is not "
                                      "supported (no recipe combines them)")
        if not 0.0 <= dc.relaxed_attention_weight <= 1.0:
            raise ValueError("relaxed_attention_weight must be in [0, 1], got %r" % (dc.relaxed_attention_weight,))
        self.cfg = cfg
        self.dictionary = dictionary
        self.register_buffer("version", torch.Tensor([3]))
        d = dc.embed_dim
        self.embed_dim = d
        self.padding_idx = embed_tokens.padding_idx
        self.max_target_positions = cfg.max_target_positions
        self.embed_tokens = embed_tokens
        self.embed_positions = _PosEmbStub()
        self.layernorm_embedding = _Affine(d) if cfg.layernorm_embedding else None
        self.layers = nn.ModuleList([_DecoderLayer(d, dc.ffn_embed_dim) for _ in range(dc.layers)])
        self.layer_norm = _Affine(d)
        self.share_input_output_embed = cfg.share_decoder_input_output_embed
        if not self.share_input_output_embed:
            self.output_projection = nn.Linear(d, len(dictionary), bias=False)
            nn.init.normal_(self.output_projection.weight, mean=0, std=d ** -0.5)
        self.engine = None
        self.flat = None
        self.dropout_seed = 2
        self.num_updates = 0
        from ..speech_lstm import ScheduledSamplingRateScheduler

        self.scheduled_sampling_rate_scheduler = ScheduledSamplingRateScheduler(
            tuple(getattr(cfg, "scheduled_sampling_probs", (1.0,))), getattr(cfg, "start_scheduled_sampling_epoch", 1))

    def flat_groups(self, prefix):
        g = []
        for i in range(len(self.layers)):
            for kind in ("weight", "bias"):
                g.append([prefix + "layers.%d.self_attn.%s_proj.%s" % (i, c, kind) for c in "qkv"])
                g.append([prefix + "layers.%d.encoder_attn.%s_proj.%s" % (i, c, kind) for c in "kv"])
        return g

    def finalize_(self, device, flat, prefix):
        self.flat = flat
        dc = self.cfg.decoder
        self.engine = DecoderEngine(flat, prefix, dict(
            embed_dim=dc.embed_dim, ffn_dim=dc.ffn_embed_dim, heads=dc.attention_heads, layers=dc.layers,
            vocab=len(self.dictionary), pad=self.padding_idx, dropout=self.cfg.dropout,
            attention_dropout=self.cfg.attention_dropout, activation_dropout=self.cfg.activation_dropout,
            layernorm_embedding=self.cfg.layernorm_embedding, share_input_output_embed=self.share_input_output_embed,
            no_scale_embedding=self.cfg.no_scale_embedding, relaxed_attention_weight=dc.relaxed_attention_weight))
        return self

    def max_positions(self):
        return self.max_target_positions

    def set_num_updates(self, n):
        self.num_updates = n

    def forward(self, prev_output_tokens, encoder_out=None, incremental_state=None, **unused):
        """Teacher-forced forward: returns (logits [B, U, V], {"attn": [None], "inner_states": [], "b200_out": ...})."""
        if incremental_state is not None:
            raise NotImplementedError("incremental decoding runs in espresso_b200 generators, not through forward()")
        from ... import ops as _ops

        enc = encoder_out["b200_out"]  # [B, T', d] batch-major
        B, U = prev_output_tokens.shape
        has_enc_pad = len(encoder_out["encoder_padding_mask"]) > 0
        enc_lens = encoder_out["src_lengths"][0].to(torch.int32) if has_enc_pad else None
        tokens = prev_output_tokens.to(torch.int32)
        tok_cpu = unused.get("prev_output_tokens_cpu")
        has_tgt_pad = bool((tok_cpu if tok_cpu is not None else prev_output_tokens).eq(self.padding_idx).any())
        tgt_lens = prev_output_tokens.ne(self.padding_idx).sum(-1).to(torch.int32) if has_tgt_pad else None
        eng = self.engine
        eng.training = self.training
        eng.seed = self.dropout_seed if _ops._SEED_T is not None else self.dropout_seed * 7919 + self.num_updates
        if torch.is_grad_enabled() and self.training:
            out = _DecoderFn.apply(enc, eng, tokens, enc_lens, tgt_lens)
        else:
            out = eng.forward(tokens, enc.detach(), enc_lens, tgt_lens, save=False)
        V = len(self.dictionary)
        return out[:, :, :V], {"attn": [None], "inner_states": [], "b200_out": out}


@register_model("speech_transformer_base", dataclass=SpeechTransformerConfig)
class SpeechTransformerModelBase(nn.Module):
    def __init__(self, cfg, encoder, decoder):
        super().__init__()
        self.cfg = cfg
        self.encoder = encoder
        self.decoder = decoder
        self.num_updates = 0
        self.frontend = None
        self.t_max_hint = 1 << 30  # generators may lower this to bound the KV caches (max decode length)

    @classmethod
    def build_embedding(cls, cfg, dictionary, embed_dim):
        emb = nn.Embedding(len(dictionary), embed_dim, padding_idx=dictionary.pad())
        nn.init.normal_(emb.weight, mean=0, std=embed_dim ** -0.5)
        nn.init.constant_(emb.weight[dictionary.pad()], 0)
        return emb

    @classmethod
    def build_model(cls, cfg, task):
        if cfg.max_source_positions is None:
            cfg.max_source_positions = DEFAULT_MAX_SOURCE_POSITIONS
        if cfg.max_target_positions is None:
            cfg.max_target_positions = DEFAULT_MAX_TARGET_POSITIONS
        e = cfg.encoder
        conv, size = ConvBNReLU.from_config(e.conv_channels, e.conv_kernel_sizes, e.conv_strides, task.feat_dim,
                                            task.feat_in_channels)
        encoder = SpeechTransformerEncoderForPrediction(cfg, pre_encoder=conv, input_size=size, vocab_size=None)
        del encoder.fc_out  # the enc-dec encoder has no output layer (keys must match the reference)
        encoder.fc_out = None
        tgt_dict = task.target_dictionary
        emb = cls.build_embedding(cfg, tgt_dict, cfg.decoder.input_dim)
        decoder = SpeechTransformerDecoderBase(cfg, tgt_dict, emb)
        return cls(cfg, encoder, decoder)

    def finalize_(self, device):
        self.to(device)
        groups = self.encoder.flat_groups("encoder.") + self.decoder.flat_groups("decoder.")
        flat = FlatParams(self, groups=groups, device=device, channels_last=self.encoder.channels_last_params("encoder."))
        self.encoder.finalize_(device, flat=flat, prefix="encoder.")
        self.decoder.finalize_(device, flat, "decoder.")
        return self

    @property
    def flat(self):
        return self.encoder.flat

    def sync_torch_grads_(self):
        self.encoder.sync_torch_grads_()

    def set_num_updates(self, n):
        self.num_updates = n
        self.encoder.set_num_updates(n)
        self.decoder.set_num_updates(n)

    def max_positions(self):
        return (self.encoder.max_positions(), self.decoder.max_positions())

    def output_lengths(self, in_lengths):
        return self.encoder.output_lengths(in_lengths)

    def forward(self, src_tokens, src_lengths, prev_output_tokens, epoch=1, freq_masks=None, time_masks=None,
                src_lengths_cpu=None, prev_output_tokens_cpu=None, time_warp=None, **kwargs):
        x, lens, lens_cpu = encoder_inputs(self, src_tokens, src_lengths, src_lengths_cpu, freq_masks, time_masks,
                                           time_warp)
        encoder_out = self.encoder(x, lens, src_lengths_cpu=lens_cpu)
        sched = getattr(self.decoder, "scheduled_sampling_rate_scheduler", None)
        if self.training and sched is not None:
            prob = sched.step(epoch)
            if prob < 1.0:
                eng = self.decoder.engine
                eng.constant_position = True  # the reference's sampled pass: every step sees the first position (see engine)
                try:
                    fed = self._scheduled_sampling_inputs(prev_output_tokens, encoder_out, prob)
                    return self.decoder(fed, encoder_out=encoder_out, prev_output_tokens_cpu=None)
                finally:
                    eng.constant_position = False
        return self.decoder(prev_output_tokens, encoder_out=encoder_out, prev_output_tokens_cpu=prev_output_tokens_cpu)

    @torch.no_grad()
    def _scheduled_sampling_inputs(self, prev_output_tokens, encoder_out, sampling_prob):
        """Scheduled sampling (espresso/models/transformer/speech_transformer_decoder.py:254-324): from step 1 on, every
        sentence feeds the TRUTH token with probability `sampling_prob` (one coin per sentence and step,
        `torch.rand([bsz, 1]).lt(p)`) and otherwise the arg-max prediction of the previous step given the tokens fed so far.
        The fed tokens carry no gradient (arg-max), and step t of the reference's incremental pass is exactly position t of a
        causal teacher-forced pass over the fed sequence (with the reference's constant position embedding, see
        DecoderEngine.constant_position; pinned against the real reference: tests/golden/scheduled_sampling.npz) -- so the
        update is: (1) this one-token-per-step pass over the incremental engine (the search kernels, no gradient; dropout
        off here, whereas the reference's predictions see its training dropout) chooses the inputs, (2) the ordinary
        forward + hand-written backward runs on them.  Rows of the padded tail are fed whatever the coin says; they only
        reach positions the loss ignores."""
        bsz, U = prev_output_tokens.shape
        dev = prev_output_tokens.device
        V = len(self.decoder.dictionary)
        state = self.init_incremental_state(encoder_out, bsz, 1)
        feed = prev_output_tokens.clone()
        buf = torch.full((bsz, U + 1), self.decoder.padding_idx, dtype=torch.int32, device=dev)
        ident = torch.arange(bsz, dtype=torch.int32, device=dev)
        pred = None
        for step in range(U):
            if step > 0:
                truth = torch.rand([bsz, 1], device=dev).lt(sampling_prob)[:, 0]
                feed[:, step] = torch.where(truth, prev_output_tokens[:, step], pred)
            buf[:, step] = feed[:, step].to(torch.int32)
            logits, _ = self.decode_step(step, buf, state, ident if step > 0 else None)
            pred = logits[:, :V].float().argmax(-1).to(prev_output_tokens.dtype)
        self.decoder.engine.training = self.training
        return feed

    def get_normalized_probs(self, net_output, log_probs, sample=None):
        logits = net_output[0].float()
        return F.log_softmax(logits, dim=-1) if log_probs else F.softmax(logits, dim=-1)

    # ---- generator protocol (espresso_b200/sequence_generator.py) --------------------------------
    def max_decoder_positions(self):
        return self.decoder.max_positions()

    def forward_encoder(self, net_input):
        x, lens, lens_cpu = encoder_inputs(self, net_input["src_tokens"], net_input["src_lengths"],
                                           net_input.get("src_lengths_cpu"))
        return self.encoder(x, lens, src_lengths_cpu=lens_cpu)

    def init_incremental_state(self, encoder_out, bsz, beam, reuse=None, attention=False):
        """attention=True: the state also records the last decoder layer's encoder attention every step (decode_attention)."""
        enc = encoder_out["b200_out"]
        has_pad = len(encoder_out["encoder_padding_mask"]) > 0
        lens = encoder_out["src_lengths"][0].to(torch.int32) if has_pad else None
        self.decoder.engine.training = False
        inc = reuse["inc"] if reuse is not None else IncrementalDecoder(self.decoder.engine)
        t_max = min(self.decoder.max_positions(), self.t_max_hint) + 2
        return {"inc": inc, "st": inc.init_state(enc, lens, bsz, beam, t_max, reuse=reuse["st"] if reuse is not None else None,
                                                 attention=attention)}

    def decode_step(self, step, tokens, state, new_order):
        return state["inc"].step(step, tokens, state["st"], new_order), True

    @staticmethod
    def advance_state_without_compute(state):
        state["inc"].advance_without_compute(state["st"])

    @staticmethod
    def decode_attention(state):
        """-> (attn fp32 [T_max, N, Tk], anc int32 [T_max, N]) after decode_step: the attention row of hypothesis n at step t
        is attn[t][anc[t][n]].  None when the state records no attention."""
        st = state["st"]
        return None if st.get("attn") is None else (st["attn"], st["anc"])


# legacy class name kept by the reference (espresso/models/transformer/speech_transformer_legacy.py:23-24)
SpeechTransformerModel = SpeechTransformerModelBase
