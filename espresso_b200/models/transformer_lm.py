"""Decoder-only Transformer language model used for shallow fusion at decode time (the `FairseqLanguageModel`
branch of espresso/speech_recognize.py:111-165; model fairseq/models/transformer_lm.py:229-323 under task
espresso/tasks/language_modeling_for_asr.py:29).  Parameter names follow fairseq's `decoder.*` keys (layers without
encoder attention).  Only incremental scoring (the generator protocol) is implemented: training the LM is an
offline step of the recipe and out of scope (SURVEY.md §2.2b)."""

import torch
import torch.nn as nn

from ..flat import FlatParams
from ..modules.decoder_engine import DecoderEngine, IncrementalDecoder
from ..registry import register_model
from .transformer.speech_transformer_encoder_model import _Affine, _Linear, _PosEmbStub
from .transformer.speech_transformer_base import _DecAttn


class _LmLayer(nn.Module):
    def __init__(self, d, ffn):
        super().__init__()
        self.self_attn = _DecAttn(d, True)
        self.self_attn_layer_norm = _Affine(d)
        self.fc1 = _Linear(d, ffn, xavier=1.0)
        self.fc2 = _Linear(ffn, d, xavier=1.0)
        self.final_layer_norm = _Affine(d)


class _LmDecoder(nn.Module):
    def __init__(self, V, d, ffn, layers, pad, share):
        super().__init__()
        self.register_buffer("version", torch.Tensor([3]))
        self.embed_tokens = nn.Embedding(V, d, padding_idx=pad)
        nn.init.normal_(self.embed_tokens.weight, mean=0, std=d ** -0.5)
        self.embed_positions = _PosEmbStub()
        self.layers = nn.ModuleList([_LmLayer(d, ffn) for _ in range(layers)])
        self.layer_norm = _Affine(d)
        if not share:
            self.output_projection = nn.Linear(d, V, bias=False)


@register_model("transformer_lm")
class TransformerLanguageModel(nn.Module):
    def __init__(self, dictionary, embed_dim=512, ffn_embed_dim=2048, layers=6, attention_heads=8, max_target_positions=1024,
                 share_decoder_input_output_embed=True):
        super().__init__()
        self.dictionary = dictionary
        self.cfg = dict(embed_dim=embed_dim, ffn_dim=ffn_embed_dim, heads=attention_heads, layers=layers, vocab=len(dictionary),
                        pad=dictionary.pad(), dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                        layernorm_embedding=False, share_input_output_embed=share_decoder_input_output_embed,
                        no_scale_embedding=False)
        self.max_target_positions = max_target_positions
        self.decoder = _LmDecoder(len(dictionary), embed_dim, ffn_embed_dim, layers, dictionary.pad(), share_decoder_input_output_embed)
        self.engine = None
        self.t_max_hint = 1 << 30

    def finalize_(self, device):
        self.to(device)
        groups = []
        for i in range(self.cfg["layers"]):
            for kind in ("weight", "bias"):
                groups.append(["decoder.layers.%d.self_attn.%s_proj.%s" % (i, c, kind) for c in "qkv"])
        self.flat = FlatParams(self, groups=groups, device=device)
        self.engine = DecoderEngine(self.flat, "decoder.", self.cfg)
        self.engine.training = False
        return self

    # ---- generator protocol ----------------------------------------------------------------------
    def max_decoder_positions(self):
        return self.max_target_positions

    def init_incremental_state(self, encoder_out, bsz, beam, reuse=None):
        inc = reuse["inc"] if reuse is not None else IncrementalDecoder(self.engine)
        t_max = min(self.max_target_positions, self.t_max_hint) + 2
        return {"inc": inc, "st": inc.init_state(None, None, bsz, beam, t_max, reuse=reuse["st"] if reuse is not None else None)}

    def decode_step(self, step, tokens, state, new_order):
        return state["inc"].step(step, tokens, state["st"], new_order), True

    @staticmethod
    def advance_state_without_compute(state):
        state["inc"].advance_without_compute(state["st"])

    # ---- prefix protocol (CTC prefix beam search: hypotheses grow on some frames only) ---------------------------
    def init_prefix_state(self, bsz, beam, T):
        """State for T frames of bsz * beam prefixes: slot 0 takes the eos context, slot f + 1 frame f's tokens.  The
        longest prefix, eos + T tokens, needs T + 2 positions (fairseq counts from padding_idx + 1)."""
        if T + 2 > self.max_target_positions:
            raise ValueError("%d encoder frames need %d LM positions, more than max_target_positions = %d"
                             % (T, T + 2, self.max_target_positions))
        inc = IncrementalDecoder(self.engine)
        return {"inc": inc, "st": inc.init_state(None, None, bsz, beam, T + 1, paths=True)}

    def prefix_step(self, slot, fed, grown, new_order, state):
        """Row n continues hypothesis new_order[n] and feeds token fed[n] (int32 [N]); it joins the prefix where grown[n].
        -> logits bf16 [N, ldV] of every row (rows that did not grow: to be discarded by the caller)."""
        return state["inc"].step(slot, fed, state["st"], new_order, grown=grown)
