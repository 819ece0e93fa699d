"""Forward / backward orchestration of the speech Transformer decoder (teacher forcing) over the sm_90a kernels.

Host-side mirror of (reference tree):
  espresso/models/transformer/speech_transformer_decoder.py:43-281
  fairseq/models/transformer/transformer_decoder.py:254-378       (embed -> layers -> layer_norm -> output proj)
  fairseq/modules/transformer_layer.py:384-533                     (pre-LN decoder block: causal self-attention,
                                                                    encoder attention, ReLU FFN)
  fairseq/modules/multihead_attention.py:639-917                   (plain scaled dot-product branch)
  fairseq/modules/sinusoidal_positional_embedding.py               (absolute positions, right-padded targets)
Activations are batch-major [B*U, d] bf16.  Like the encoder engine this only sequences kernel calls and owns the
saved-for-backward tensors; the backward is written by hand and accumulates into the flat fp32 gradient buffer.
"""
import math

import torch

from .. import ops as _ops
from ..lib import ACT_RELU, ACT_RELU_BWD
from .encoder_engine import LN_EPS, EncoderEngine, _r8, sinusoidal_positions


class DecoderEngine(EncoderEngine):
    _FFN = ("final_layer_norm", "fc1", "fc2")

    def __init__(self, flat, prefix, cfg):
        """cfg keys: embed_dim, ffn_dim, heads, layers, vocab, pad, dropout, attention_dropout, activation_dropout,
        layernorm_embedding, share_input_output_embed, no_scale_embedding, relaxed_attention_weight (encoder attention,
        training only; default 0)."""
        super().__init__(flat, prefix, dict(cfg, layer_type="decoder"))
        self._pos = {}
        # Scheduled sampling in the reference feeds a [B, 1] token tensor per step, so its sinusoidal position module
        # (incremental branch, fairseq/modules/sinusoidal_positional_embedding.py:78-87: pos = seq_len = 1) gives EVERY
        # step the embedding of the first position; the model sets this flag for such updates to reproduce it.
        self.constant_position = False

    def positions(self, U, device):
        key = (U, str(device), self.constant_position)
        if key not in self._pos:
            tab = sinusoidal_positions(U, self.d, self.cfg["pad"], device)
            self._pos[key] = tab[:1].expand(U, -1).contiguous() if self.constant_position else tab
        return self._pos[key]

    # ---- causal self-attention -------------------------------------------------------------------
    def self_attn_fwd(self, x, lp, B, U, tgt_lens, li):
        d = self.d
        ln, mean, rstd = _ops.layer_norm_fwd(x, self.P(lp + "self_attn_layer_norm.weight"),
                                             self.P(lp + "self_attn_layer_norm.bias"), LN_EPS)
        W, b, _, _ = self._proj(lp, "self_attn", "qkv")
        qkv = _ops.linear(ln, W, b)
        ctx, att = self._attend(qkv[:, :d], 3 * d, qkv[:, d:2 * d], qkv[:, 2 * d:], 3 * d, B, U, U, tgt_lens, True, li, 30)
        y = _ops.linear(ctx, self.P(lp + "self_attn.out_proj.weight"), self.P(lp + "self_attn.out_proj.bias"),
                        drop_p=self._drop("dropout"), drop_mode=1, seed=self._seed(li, 31), R=x, ldr=x.stride(0), beta=1.0)
        return y, (x, mean, rstd, ln, qkv, att, ctx)

    def self_attn_bwd(self, dy, saved, lp, B, U, li):
        d = self.d
        x, mean, rstd, ln, qkv, att, ctx = saved
        dO = _ops.dropout(dy, self._drop("dropout"), self._seed(li, 31))
        _ops.linear_wgrad(dO, ctx, self.G(lp + "self_attn.out_proj.weight"), self.G(lp + "self_attn.out_proj.bias"))
        dctx = _ops.linear_dgrad(dO, self.P(lp + "self_attn.out_proj.weight"))
        dqkv = torch.empty_like(qkv)
        self._attend_bwd(dctx, att, qkv[:, :d], 3 * d, qkv[:, d:2 * d], qkv[:, 2 * d:], 3 * d, dqkv[:, :d], 3 * d,
                         dqkv[:, d:2 * d], dqkv[:, 2 * d:], 3 * d, B, U, U, li, 30)
        W, _, gW, gb = self._proj(lp, "self_attn", "qkv")
        _ops.linear_wgrad(dqkv, ln, gW, gb)
        dln = _ops.linear_dgrad(dqkv, W)
        return _ops.layer_norm_bwd(dln, x, mean, rstd, self.P(lp + "self_attn_layer_norm.weight"),
                                   self.G(lp + "self_attn_layer_norm.weight"), self.G(lp + "self_attn_layer_norm.bias"), dres=dy)

    # ---- encoder (cross) attention -----------------------------------------------------------------
    def cross_attn_fwd(self, x, enc, lp, B, U, Tk, enc_lens, li):
        d = self.d
        ln, mean, rstd = _ops.layer_norm_fwd(x, self.P(lp + "encoder_attn_layer_norm.weight"),
                                             self.P(lp + "encoder_attn_layer_norm.bias"), LN_EPS)
        q = _ops.linear(ln, self.P(lp + "encoder_attn.q_proj.weight"), self.P(lp + "encoder_attn.q_proj.bias"))
        Wkv, bkv, _, _ = self._proj(lp, "encoder_attn", "kv")
        kv = _ops.linear(enc, Wkv, bkv)  # [B*Tk, 2d]
        # relaxed encoder attention in training (multihead_attention.py:869-872): w / Tk with Tk the padded length
        relax = float(self.cfg.get("relaxed_attention_weight", 0.0)) if self.training else 0.0
        ctx, att = self._attend(q, d, kv[:, :d], kv[:, d:], 2 * d, B, U, Tk, enc_lens, False, li, 32, relax=relax)
        y = _ops.linear(ctx, self.P(lp + "encoder_attn.out_proj.weight"), self.P(lp + "encoder_attn.out_proj.bias"),
                        drop_p=self._drop("dropout"), drop_mode=1, seed=self._seed(li, 33), R=x, ldr=x.stride(0), beta=1.0)
        return y, (x, mean, rstd, ln, q, kv, att, ctx)

    def cross_attn_bwd(self, dy, saved, enc, denc, lp, B, U, Tk, li):
        d = self.d
        x, mean, rstd, ln, q, kv, att, ctx = saved
        dO = _ops.dropout(dy, self._drop("dropout"), self._seed(li, 33))
        _ops.linear_wgrad(dO, ctx, self.G(lp + "encoder_attn.out_proj.weight"), self.G(lp + "encoder_attn.out_proj.bias"))
        dctx = _ops.linear_dgrad(dO, self.P(lp + "encoder_attn.out_proj.weight"))
        dq = torch.empty_like(q)
        dkv = torch.empty_like(kv)
        self._attend_bwd(dctx, att, q, d, kv[:, :d], kv[:, d:], 2 * d, dq, d, dkv[:, :d], dkv[:, d:], 2 * d, B, U, Tk, li, 32)
        Wkv, _, gWkv, gbkv = self._proj(lp, "encoder_attn", "kv")
        _ops.linear_wgrad(dkv, enc, gWkv, gbkv)
        # gradient w.r.t. the encoder output accumulates over decoder layers: denc += dkv @ Wkv
        _ops.linear_dgrad(dkv, Wkv, out=denc, R=denc, ldr=d, beta=1.0)
        _ops.linear_wgrad(dq, ln, self.G(lp + "encoder_attn.q_proj.weight"), self.G(lp + "encoder_attn.q_proj.bias"))
        dln = _ops.linear_dgrad(dq, self.P(lp + "encoder_attn.q_proj.weight"))
        return _ops.layer_norm_bwd(dln, x, mean, rstd, self.P(lp + "encoder_attn_layer_norm.weight"),
                                   self.G(lp + "encoder_attn_layer_norm.weight"), self.G(lp + "encoder_attn_layer_norm.bias"),
                                   dres=dy)

    # ---- whole decoder ------------------------------------------------------------------------------
    def out_weight(self):
        return self.P("embed_tokens.weight") if self.cfg.get("share_input_output_embed", False) else self.P("output_projection.weight")

    def out_grad(self):
        return self.G("embed_tokens.weight") if self.cfg.get("share_input_output_embed", False) else self.G("output_projection.weight")

    def forward(self, tokens, enc, enc_lens, tgt_lens, save=True):
        """tokens int32 [B, U] (prev_output_tokens, right padded); enc bf16 [B, Tk, d], or None for a language model's
        layers (no encoder attention; forward only); enc_lens int32 [B] or None (no encoder padding); tgt_lens int32 [B]
        or None (no target padding).  Returns logits [B, U, ldV]."""
        cfg = self.cfg
        B, U = tokens.shape
        Tk = enc.shape[1] if enc is not None else 0
        d, V = self.d, cfg["vocab"]
        scale = 1.0 if cfg.get("no_scale_embedding", False) else math.sqrt(d)
        tok = tokens.reshape(-1).contiguous()
        pdrop = self._drop("dropout")
        lne = cfg.get("layernorm_embedding", False)
        x = _ops.embed_fwd(tok, self.P("embed_tokens.weight"), self.positions(U, tokens.device), U, scale, cfg["pad"],
                           0.0 if lne else pdrop, self._seed(998, 0))
        emb = None
        if lne:
            emb = x
            x, m0, r0 = _ops.layer_norm_fwd(emb, self.P("layernorm_embedding.weight"), self.P("layernorm_embedding.bias"), LN_EPS,
                                            drop_p=pdrop, seed=self._seed(998, 0))
            emb = (emb, m0, r0)
        enc2 = enc.reshape(B * Tk, d) if enc is not None else None
        states = []
        for li in range(cfg["layers"]):
            lp = "layers.%d." % li
            st = {}
            x, st["self"] = self.self_attn_fwd(x, lp, B, U, tgt_lens, li)
            if enc is not None:
                x, st["cross"] = self.cross_attn_fwd(x, enc2, lp, B, U, Tk, enc_lens, li)
            x, st["ffn"] = self.ffn_fwd(x, lp, self._FFN, ACT_RELU, 1.0, li, 34)
            states.append(st)
        xf = x
        x, mf, rf = _ops.layer_norm_fwd(xf, self.P("layer_norm.weight"), self.P("layer_norm.bias"), LN_EPS)
        ldV = _r8(V)
        R = B * U
        logits = torch.zeros(R, ldV, device=x.device, dtype=torch.bfloat16) if ldV != V else \
            torch.empty(R, ldV, device=x.device, dtype=torch.bfloat16)
        W = self.out_weight()
        _ops.gemm(x, W, logits, R, V, d, d, W.stride(0), ldV)
        if save and enc is not None:
            self.saved = dict(B=B, U=U, Tk=Tk, tok=tok, emb=emb, enc2=enc2, states=states, fin=(xf, mf, rf), xL=x, scale=scale)
        return logits.view(B, U, ldV)

    def backward(self, dlogits):
        """dlogits [B, U, ldV] -> d(enc) [B, Tk, d]; parameter gradients go to the flat buffer."""
        s = self.saved
        cfg = self.cfg
        B, U, Tk, d, V = s["B"], s["U"], s["Tk"], self.d, cfg["vocab"]
        R = B * U
        ldV = _r8(V)
        dlog = dlogits.reshape(R, ldV)
        dl = dlog[:, :V] if ldV != V else dlog
        _ops.linear_wgrad(dl, s["xL"], self.out_grad())
        dx = _ops.linear_dgrad(dl, self.out_weight())
        xf, mf, rf = s["fin"]
        dx = _ops.layer_norm_bwd(dx, xf, mf, rf, self.P("layer_norm.weight"), self.G("layer_norm.weight"), self.G("layer_norm.bias"))
        denc = torch.zeros(B * Tk, d, device=dx.device, dtype=torch.bfloat16)
        for li in reversed(range(cfg["layers"])):
            lp = "layers.%d." % li
            st = s["states"][li]
            dx = self.ffn_bwd(dx, st["ffn"], lp, self._FFN, ACT_RELU_BWD, 1.0, li, 34)
            dx = self.cross_attn_bwd(dx, st["cross"], s["enc2"], denc, lp, B, U, Tk, li)
            dx = self.self_attn_bwd(dx, st["self"], lp, B, U, li)
        pdrop = self._drop("dropout")
        if s["emb"] is not None:
            e, m0, r0 = s["emb"]
            dx = _ops.layer_norm_bwd(dx, e, m0, r0, self.P("layernorm_embedding.weight"), self.G("layernorm_embedding.weight"),
                                     self.G("layernorm_embedding.bias"), drop_p=pdrop, seed=self._seed(998, 0))
            pdrop = 0.0
        _ops.embed_bwd(s["tok"], dx, self.G("embed_tokens.weight"), s["scale"], cfg["pad"], pdrop, self._seed(998, 0))
        self.saved = None
        return denc.view(B, Tk, d)


class IncrementalDecoder:
    """One-token-per-hypothesis decoder step for beam search (eval only), over the same flat parameters as
    DecoderEngine.  Mirrors the incremental branch of the reference decoder
    (fairseq/models/transformer/transformer_decoder.py:300-305 `prev_output_tokens[:, -1:]`,
    fairseq/modules/transformer_layer.py:384-533 with incremental_state, multihead_attention.py:639-760).

    State: per layer a K/V cache [T_max, N, 2d] written in place by the K/V projection GEMM, an ancestry table
    [T_max, N] (see csrc/decode_attn.cu) and the encoder-attention K/V [bsz, Tk, 2d] computed once per sentence
    (the reference's beamable encoder attention, multihead_attention.py:661-669).  With attention=True it also keeps
    "attn" [T_max, N, Tk] fp32: row (t, r) = the last layer's head-averaged encoder attention of cache row r at step t
    (transformer_decoder.py:283-284), indexed like the K/V cache, so beam reordering never moves it either.

    Prefix-state mode (init_state(..., paths=True); language model only): hypotheses grow on different steps, as the
    prefixes of a CTC prefix beam search do.  The K/V cache [S, N, 2d] is then indexed by SLOT (step s writes slot s for
    every row; slot 0 holds the eos context) and each hypothesis keeps a path table instead of an ancestry table:
    "cells" [S, N] = the flat cells slot * N + row of its keys and "len" [N] = their count (esp_decode_update_paths).  A
    hypothesis of length L feeds its next token at position L."""

    def __init__(self, engine: DecoderEngine):
        self.e = engine

    def init_state(self, enc, enc_lens, bsz, beam, t_max, reuse=None, attention=False, paths=False):
        """enc bf16 [bsz, Tk, d] or None (language model: no encoder attention).  paths: prefix-state mode (enc None, no
        reuse), t_max slots; every path starts empty.

        `reuse`: a state returned earlier for the SAME shapes -- its buffers are re-initialised in place (KV caches keep
        their addresses, ancestry tables are zeroed and put back in their initial roles, the encoder-attention K/V are
        recomputed into the same tensors), which is what lets a search step be replayed from a CUDA graph."""
        e = self.e
        d, Lr = e.d, e.cfg["layers"]
        N = bsz * beam
        dev = e.flat.p16.device
        Tk = enc.shape[1] if enc is not None else 0
        attention = attention and enc is not None
        sig = (N, beam, bsz, t_max, Tk, enc_lens is not None, attention)
        if paths:
            assert enc is None and reuse is None
            st = dict(N=N, beam=beam, bsz=bsz, t_max=t_max, paths=True, cross=None, attn=None)
            st["kv"] = [torch.empty(t_max, N, 2 * d, device=dev, dtype=torch.bfloat16) for _ in range(Lr)]
            st["cells"], st["cells_alt"] = (torch.zeros(t_max, N, device=dev, dtype=torch.int32) for _ in range(2))
            st["len"], st["len_alt"] = (torch.zeros(N, device=dev, dtype=torch.int32) for _ in range(2))
            st["pos_idx"] = torch.empty(N, device=dev, dtype=torch.int32)
            return st
        if reuse is not None and reuse.get("sig") == sig:
            st = reuse
            st["anc"], st["anc_alt"] = st["anc0"], st["anc1"]
            st["anc"].zero_()
            st["anc_alt"].zero_()
            if enc_lens is not None:
                st["enc_lens"].copy_(enc_lens)
        else:
            st = dict(N=N, beam=beam, bsz=bsz, t_max=t_max, sig=sig)
            st["enc_lens"] = enc_lens.clone() if enc_lens is not None else None
            st["kv"] = [torch.empty(t_max, N, 2 * d, device=dev, dtype=torch.bfloat16) for _ in range(Lr)]
            st["anc0"] = torch.zeros(t_max, N, device=dev, dtype=torch.int32)
            st["anc1"] = torch.zeros_like(st["anc0"])
            st["anc"], st["anc_alt"] = st["anc0"], st["anc1"]
            st["cross"] = [torch.empty(bsz, Tk, 2 * d, device=dev, dtype=torch.bfloat16) for _ in range(Lr)] if enc is not None else None
            st["attn"] = torch.empty(t_max, N, Tk, device=dev, dtype=torch.float32) if attention else None
        if enc is not None:
            enc2 = enc.reshape(bsz * Tk, d)
            for li in range(Lr):
                Wkv, bkv, _, _ = e._proj("layers.%d." % li, "encoder_attn", "kv")
                _ops.linear(enc2, Wkv, bkv, out=st["cross"][li].view(bsz * Tk, 2 * d))
        return st

    @staticmethod
    def advance_without_compute(st):
        """Host-side effect of step() when its device work is replayed from a CUDA graph: the ancestry tables swap."""
        st["anc"], st["anc_alt"] = st["anc_alt"], st["anc"]

    def step(self, step, tokens, st, new_order, grown=None):
        """tokens int32 [N, L] (column `step` is the newest token) -> logits bf16 [N, ldV].

        Prefix-state mode: `step` is the slot, tokens int32 [N] the token each row feeds, new_order int32 [N] the row
        each hypothesis continues and grown int32 [N] whether its fed token joins its prefix (a row that did not grow
        still computes, at its current length; its logits are for the caller to discard)."""
        e = self.e
        cfg = e.cfg
        d, H, V = e.d, e.H, cfg["vocab"]
        N = st["N"]
        if st.get("paths"):
            _ops.decode_update_paths(st["cells"], st["len"], st["cells_alt"], st["len_alt"], new_order, grown, step,
                                     pos_out=st["pos_idx"])
            st["cells"], st["cells_alt"], st["len"], st["len_alt"] = st["cells_alt"], st["cells"], st["len_alt"], st["len"]
            tok = tokens
            pos, U = _ops.gather_rows(e.positions(st["t_max"], tokens.device), st["pos_idx"]), N
            attend = lambda q, kv: _ops.decode_self_attn_paths(q, kv, st["cells"], st["len"], H, e.scaling)  # noqa: E731
        else:
            _ops.decode_update_ancestry(st["anc"], st["anc_alt"], new_order if step > 0 else None, step)
            st["anc"], st["anc_alt"] = st["anc_alt"], st["anc"]
            tok = tokens[:, step].contiguous()
            pos, U = e.positions(st["t_max"], tokens.device)[step: step + 1], 1
            attend = lambda q, kv: _ops.decode_self_attn(q, kv, st["anc"], step + 1, H, e.scaling)  # noqa: E731
        scale = 1.0 if cfg.get("no_scale_embedding", False) else math.sqrt(d)
        x = _ops.embed_fwd(tok, e.P("embed_tokens.weight"), pos, U, scale, cfg["pad"])
        if cfg.get("layernorm_embedding", False):
            x, _, _ = _ops.layer_norm_fwd(x, e.P("layernorm_embedding.weight"), e.P("layernorm_embedding.bias"), LN_EPS)
        for li in range(cfg["layers"]):
            lp = "layers.%d." % li
            ln, _, _ = _ops.layer_norm_fwd(x, e.P(lp + "self_attn_layer_norm.weight"), e.P(lp + "self_attn_layer_norm.bias"), LN_EPS)
            W, b, _, _ = e._proj(lp, "self_attn", "qkv")
            q = _ops.linear(ln, W[:d], b[:d])
            _ops.linear(ln, W[d:], b[d:], out=st["kv"][li][step])  # K | V of this step, written into the cache
            ctx = attend(q, st["kv"][li])
            x = _ops.linear(ctx, e.P(lp + "self_attn.out_proj.weight"), e.P(lp + "self_attn.out_proj.bias"), R=x, ldr=d, beta=1.0)
            if st["cross"] is not None:
                ln, _, _ = _ops.layer_norm_fwd(x, e.P(lp + "encoder_attn_layer_norm.weight"), e.P(lp + "encoder_attn_layer_norm.bias"),
                                               LN_EPS)
                q = _ops.linear(ln, e.P(lp + "encoder_attn.q_proj.weight"), e.P(lp + "encoder_attn.q_proj.bias"))
                if st["attn"] is not None and li == cfg["layers"] - 1:
                    ctx = _ops.decode_cross_attn_weights(q, st["cross"][li], st["enc_lens"], st["beam"], H, e.scaling, st["attn"][step])
                else:
                    ctx = _ops.decode_cross_attn(q, st["cross"][li], st["enc_lens"], st["beam"], H, e.scaling)
                x = _ops.linear(ctx, e.P(lp + "encoder_attn.out_proj.weight"), e.P(lp + "encoder_attn.out_proj.bias"), R=x, ldr=d,
                                beta=1.0)
            ln, _, _ = _ops.layer_norm_fwd(x, e.P(lp + "final_layer_norm.weight"), e.P(lp + "final_layer_norm.bias"), LN_EPS)
            hh = _ops.linear(ln, e.P(lp + "fc1.weight"), e.P(lp + "fc1.bias"), act=ACT_RELU)
            x = _ops.linear(hh, e.P(lp + "fc2.weight"), e.P(lp + "fc2.bias"), R=x, ldr=d, beta=1.0)
        x, _, _ = _ops.layer_norm_fwd(x, e.P("layer_norm.weight"), e.P("layer_norm.bias"), LN_EPS)
        ldV = _r8(V)
        logits = torch.empty(N, ldV, device=x.device, dtype=torch.bfloat16)
        Wo = e.out_weight()
        _ops.gemm(x, Wo, logits, N, V, d, d, Wo.stride(0), ldV)
        return logits
