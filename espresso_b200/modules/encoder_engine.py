"""Forward / backward orchestration of the speech Transformer/Conformer encoder over the sm_90a kernels.

This is the host-side mirror of (paths in the reference tree):
  espresso/models/transformer/speech_transformer_encoder.py:298-409   (fc0, layernorm_embedding, layer loop)
  espresso/modules/conformer_with_relative_positional_embedding_encoder_layer.py:81-145   (Conformer block)
  fairseq/modules/conformer_layer.py:79-101,134-146                     (conv module, feed-forward module)
  fairseq/modules/multihead_attention.py:639-917                        (relative-position / plain self-attention)
  fairseq/modules/sinusoidal_positional_embedding.py                    (absolute positions, padding_idx 0)
  fairseq/modules/transformer_layer.py:163-226                          (pre-LN Transformer block)
  espresso/models/transformer/speech_transformer_encoder_model.py:177-210 (fc_out)
Activations are batch-major [B*T, d] bf16.  Every arithmetic step is one call into libespresso_b200.so
(`ops`); this file only sequences them, owns the saved-for-backward tensors and hands the kernels views
of the flat parameter / gradient buffers.  The backward pass is written by hand (no autograd tape): each
module's backward mirrors its forward line by line and accumulates parameter gradients directly into
the flat fp32 gradient buffer.
"""
import math
import os

import torch

from .. import ops as _ops
from ..lib import ACT_RELU, ACT_RELU_BWD, ACT_SILU, ACT_SILU_BWD

LN_EPS = 1e-5
BN_EPS = 1e-5
BN_MOMENTUM = 0.1


def _r8(n):
    return (n + 7) // 8 * 8


def sinusoidal_relative_table(T, d, device, dtype=torch.bfloat16):
    """Rows for relative positions -(T-1)..(T-1), scaled by d^-0.5 (scale_embedding=True), sin | cos halves.

    espresso/modules/sinusoidal_relative_positional_embedding.py:46-71,73-124 and
    espresso/modules/relative_positional_embedding.py:28-34.  Computed in fp32 then cast to the model
    dtype exactly like `self.weight.to(self._float_tensor)`."""
    half = d // 2
    freq = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000.0) / (half - 1)))
    pos = torch.arange(-(T - 1), T, dtype=torch.float32)[:, None] * freq[None, :]
    emb = torch.cat([torch.sin(pos), torch.cos(pos)], dim=1)
    if d % 2 == 1:
        emb = torch.cat([emb, torch.zeros(emb.shape[0], 1)], dim=1)
    return (emb * d ** -0.5).to(device=device, dtype=dtype).contiguous()


def sinusoidal_positions(U, d, padding_idx, device, dtype=torch.bfloat16):
    """Rows t = 0..U-1 of fairseq's sinusoidal table at index t + padding_idx + 1 (right-padded sequences),
    computed in fp32 then cast to the model dtype."""
    half = d // 2
    f = torch.exp(torch.arange(half, dtype=torch.float) * -(math.log(10000) / (half - 1)))
    pos = torch.arange(padding_idx + 1, padding_idx + 1 + U, dtype=torch.float)[:, None] * f[None, :]
    e = torch.cat([torch.sin(pos), torch.cos(pos)], dim=1)
    if d % 2 == 1:
        e = torch.cat([e, torch.zeros(U, 1)], dim=1)
    return e.to(device=device, dtype=dtype).contiguous()


class EncoderEngine:
    def __init__(self, flat, prefix, cfg):
        """cfg keys: embed_dim, ffn_dim, heads, layers, layer_type ('conformer'|'transformer'), dw_kernel,
        dropout, attention_dropout, activation_dropout, layernorm_embedding, final_layer_norm, vocab (or None),
        learned_pos_tables (None, or {layer index: flat parameter name of that layer's learned relative-position
        table} -- shared tables map several layers to one name), rel_pos (default True; False: sinusoidal absolute positions
        added after fc0 and plain scaled dot-product self-attention)."""
        self.flat = flat
        self.pre = prefix
        self.cfg = dict(cfg)
        self.d = cfg["embed_dim"]
        self.H = cfg["heads"]
        self.hd = self.d // self.H
        self.scaling = self.hd ** -0.5
        self._pe = {}
        self._zeros_d = None
        self.pos_tables = cfg.get("learned_pos_tables")  # espresso/modules/learned_relative_positional_embedding.py
        self.rel_pos = cfg.get("rel_pos", True)
        self.bn_state = None  # {layer: (running_mean fp32, running_var fp32)} provided by the module
        self.training = True
        self.seed = 0
        # rel-pos attention forward as one fused wgmma kernel (csrc/attn_fused.cu); ESP_FUSED_ATTN=0 restores the
        # round-1 chain (BD GEMM -> QK^T+skew GEMM -> softmax -> P V GEMM) for A/B comparisons
        self.fused_attention = os.environ.get("ESP_FUSED_ATTN", "1") != "0"
        # ... and the score side of its backward (csrc/attn_fused_bwd.cu); ESP_FUSED_ATTN_BWD=0 keeps the unfused chain
        self.fused_attention_bwd = os.environ.get("ESP_FUSED_ATTN_BWD", "1") != "0"
        self._save_probs = True
        self.key_bounds = None  # (lo, hi) int32 [T] device tensors: per-row visible key range (streaming masks)

    # ------------------------------------------------------------------------------------------
    def P(self, name):
        return self.flat.param(self.pre + name)

    def G(self, name):
        return self.flat.grad(self.pre + name)

    def _qkv(self, lp):
        names = [self.pre + lp + "self_attn.%s_proj.weight" % c for c in "qkv"]
        bn = [self.pre + lp + "self_attn.%s_proj.bias" % c for c in "qkv"]
        d = self.d
        return (self.flat.span(self.flat.p16, names, (3 * d, d)), self.flat.span(self.flat.p16, bn, (3 * d,)),
                self.flat.span(self.flat.g32, names, (3 * d, d)), self.flat.span(self.flat.g32, bn, (3 * d,)))

    def pe(self, T, device):
        key = (T, str(device))
        if key not in self._pe:
            self._pe[key] = sinusoidal_relative_table(T, self.d, device)
        return self._pe[key]

    def abs_pe(self, T, device):
        """Absolute positions of frames 0..T-1 (speech_transformer_encoder.py:93-101,343-345): fairseq's sinusoidal table
        with padding_idx 0 indexed by the non-padding mask, i.e. row t + 1 for a valid frame t and the zero row for a padded
        one.  Every frame gets row t + 1 here: padded rows are zeroed right after (layernorm_embedding with lens, or
        mask_rows) and LayerNorm is per row, so what a padded row held before that never reaches a valid one -- and the
        gradient of those rows is zeroed the same way in the backward pass."""
        key = ("abs", T, str(device))
        if key not in self._pe:
            self._pe[key] = sinusoidal_positions(T, self.d, 0, device)
        return self._pe[key]

    def _learned_positions(self, li, T, device):
        """Rows of layer li's learned table for relative positions -(T-1)..T-1 (learned_relative_positional_embedding.py
        :71-78: start = n/2 - T + 1, clamped when T > max_size).  Returns (pe [2T-1, E] bf16, index tensor)."""
        name = self.pos_tables[li]
        tab = self.flat.param(name)
        n = tab.shape[0]
        key = ("pos", T, n, str(device))
        if key not in self._pe:
            self._pe[key] = torch.arange(n // 2 - T + 1, n // 2 + T, device=device).clamp_(0, n - 1)
        idx = self._pe[key]
        return tab.index_select(0, idx), idx

    def _drop(self, kind):
        if not self.training:
            return 0.0
        return float(self.cfg.get(kind, 0.0))

    def _seed(self, layer, op):
        return (self.seed * 1000003 + layer * 64 + op) & 0x7FFFFFFFFFFFFFFF

    # ---- feed-forward module ----------------------------------------------------------------------
    def ffn_fwd(self, x, lp, names, act, alpha, li, opbase):
        ln_n, w1_n, w2_n = names
        ln, mean, rstd = _ops.layer_norm_fwd(x, self.P(lp + ln_n + ".weight"), self.P(lp + ln_n + ".bias"), LN_EPS)
        W1, W2 = self.P(lp + w1_n + ".weight"), self.P(lp + w2_n + ".weight")
        R = x.shape[0]
        U = torch.empty(R, W1.shape[0], device=x.device, dtype=torch.bfloat16)
        Hh = _ops.linear(ln, W1, self.P(lp + w1_n + ".bias"), act=act, C2=U, drop_p=self._drop("activation_dropout"),
                         drop_mode=1, seed=self._seed(li, opbase))
        y = _ops.linear(Hh, W2, self.P(lp + w2_n + ".bias"), drop_p=self._drop("dropout"), drop_mode=1,
                        seed=self._seed(li, opbase + 1), alpha=alpha, R=x, ldr=x.stride(0), beta=1.0)
        return y, (x, mean, rstd, ln, U, Hh)

    def ffn_bwd(self, dy, saved, lp, names, act_bwd, alpha, li, opbase, dyd=None, next_drop=None):
        """dyd: dropout(dy) * alpha already formed by the previous module's LayerNorm backward (same mask stream);
        next_drop: (p, seed, scale) of the module whose backward runs next -- its masked gradient is returned as a
        second value (written by this module's LayerNorm backward instead of by a separate dropout pass)."""
        ln_n, w1_n, w2_n = names
        x, mean, rstd, ln, U, Hh = saved
        W1, W2 = self.P(lp + w1_n + ".weight"), self.P(lp + w2_n + ".weight")
        dZ = dyd if dyd is not None else _ops.dropout(dy, self._drop("dropout"), self._seed(li, opbase + 1), scale=alpha)
        _ops.linear_wgrad(dZ, Hh, self.G(lp + w2_n + ".weight"), self.G(lp + w2_n + ".bias"))
        dU = _ops.linear_dgrad(dZ, W2, act=act_bwd, aux=U, ld_aux=U.stride(0), drop_p=self._drop("activation_dropout"),
                               drop_mode=2, seed=self._seed(li, opbase))
        _ops.linear_wgrad(dU, ln, self.G(lp + w1_n + ".weight"), self.G(lp + w1_n + ".bias"))
        dln = _ops.linear_dgrad(dU, W1)
        return _ops.layer_norm_bwd(dln, x, mean, rstd, self.P(lp + ln_n + ".weight"), self.G(lp + ln_n + ".weight"),
                                   self.G(lp + ln_n + ".bias"), dres=dy, next_drop=next_drop)

    # ---- relative-position multi-head self-attention ---------------------------------------------
    def mha_fwd(self, x, lp, B, T, lens, li):
        d, H, hd = self.d, self.H, self.hd
        R = B * T
        ln, mean, rstd = _ops.layer_norm_fwd(x, self.P(lp + "self_attn_layer_norm.weight"),
                                             self.P(lp + "self_attn_layer_norm.bias"), LN_EPS)
        Wqkv, bqkv, _, _ = self._qkv(lp)
        qkv = _ops.linear(ln, Wqkv, bqkv)
        q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        if not self.rel_pos:
            ctx, att = self._plain_attn_fwd(q, k, v, B, T, lens, li)
            y = _ops.linear(ctx, self.P(lp + "self_attn.out_proj.weight"), self.P(lp + "self_attn.out_proj.bias"),
                            drop_p=self._drop("dropout"), drop_mode=1, seed=self._seed(li, 11), R=x, ldr=x.stride(0), beta=1.0)
            return y, (x, mean, rstd, ln, qkv, att, ctx)
        learned = self.pos_tables is not None
        if learned:
            # learned relative positions: q is only scaled (no pos_bias_u / pos_bias_v), the table rows are used as they
            # are (no pos_proj); a table of width head_dim is shared by all heads (head stride 0 in the GEMM)
            if self._zeros_d is None or self._zeros_d.device != x.device:
                self._zeros_d = torch.zeros(d, device=x.device, dtype=torch.bfloat16)
            qu, _unused = _ops.qprep_fwd(q, self._zeros_d, self._zeros_d, self.scaling)
            qv = qu
            Pp, _ = self._learned_positions(li, T, x.device)
        else:
            qu, qv = _ops.qprep_fwd(q, self.P(lp + "self_attn.pos_bias_u"), self.P(lp + "self_attn.pos_bias_v"), self.scaling)
            pe = self.pe(T, x.device)
            Pp = _ops.linear(pe, self.P(lp + "self_attn.pos_proj.weight"))  # [2T-1, d], batch independent
        E = Pp.shape[1]
        ph = hd if E == d else 0  # head stride of the position operand
        if self.fused_attention and hd == 64:
            # scores, relative-position logits, skew, softmax and P v in ONE kernel (csrc/attn_fused.cu); only the
            # probabilities the backward pass needs go to HBM
            ctx, Pr, Pd = _ops.attn_fused_fwd(qu, qv, k, v, Pp, B, T, H, lens, self._drop("attention_dropout"),
                                              self._seed(li, 10), save_probs=self._save_probs, pos_hstride=ph,
                                              key_bounds=self.key_bounds)
        else:
            if self.key_bounds is not None:
                raise NotImplementedError("chunk-streaming / limited-context masks run in the fused attention kernel only "
                                          "(head_dim 64, ESP_FUSED_ATTN unset)")
            ldt, ldp = _r8(T), _r8(2 * T - 1)
            BD = torch.empty(H, B, T, ldp, device=x.device, dtype=torch.bfloat16)
            _ops.gemm(qv, Pp, BD, T, 2 * T - 1, hd, d, E, ldp, nb1=H, nb2=B, sA=(hd, T * d), sB=(ph, 0),
                      sC=(B * T * ldp, T * ldp))
            S = torch.empty(H, B, T, ldt, device=x.device, dtype=torch.bfloat16)
            _ops.gemm(qu, k, S, T, T, hd, d, 3 * d, ldt, nb1=H, nb2=B, sA=(hd, T * d), sB=(hd, T * 3 * d),
                      sC=(B * T * ldt, T * ldt), R=BD, ldr=ldp, sR=(B * T * ldp, T * ldp), skew_r=T)
            Pr, Pd = _ops.attn_softmax_fwd(S, T, lens, self._drop("attention_dropout"), self._seed(li, 10))
            ctx = torch.empty(R, d, device=x.device, dtype=torch.bfloat16)
            _ops.gemm(Pd, v, ctx, T, hd, T, ldt, 3 * d, d, b_kmajor=False, nb1=H, nb2=B, sA=(B * T * ldt, T * ldt),
                      sB=(hd, T * 3 * d), sC=(hd, T * d))
        y = _ops.linear(ctx, self.P(lp + "self_attn.out_proj.weight"), self.P(lp + "self_attn.out_proj.bias"),
                        drop_p=self._drop("dropout"), drop_mode=1, seed=self._seed(li, 11), R=x, ldr=x.stride(0), beta=1.0)
        return y, (x, mean, rstd, ln, qkv, qu, qv, Pp, Pr, Pd, ctx)

    def mha_bwd(self, dy, saved, lp, B, T, li, dyd=None, next_drop=None):
        if not self.rel_pos:
            return self._plain_mha_bwd(dy, saved, lp, B, T, li, dyd, next_drop)
        d, H, hd = self.d, self.H, self.hd
        R = B * T
        x, mean, rstd, ln, qkv, qu, qv, Pp, Pr, Pd, ctx = saved
        k, v = qkv[:, d:2 * d], qkv[:, 2 * d:]
        ldt, ldp = _r8(T), _r8(2 * T - 1)
        dev = dy.device
        dO = dyd if dyd is not None else _ops.dropout(dy, self._drop("dropout"), self._seed(li, 11))
        _ops.linear_wgrad(dO, ctx, self.G(lp + "self_attn.out_proj.weight"), self.G(lp + "self_attn.out_proj.bias"))
        dctx = _ops.linear_dgrad(dO, self.P(lp + "self_attn.out_proj.weight"))
        dqkv = torch.empty(R, 3 * d, device=dev, dtype=torch.bfloat16)
        dqu = torch.empty(R, d, device=dev, dtype=torch.bfloat16)
        if self.fused_attention and hd == 64 and self.fused_attention_bwd and T <= 1024:  # skew kernel: rows of <= 1024 keys
            # ONE kernel: dPd = dctx v^T in registers, dS in registers (written once, plain and skewed), dV = Pd^T dctx and
            # dK = dS^T q_u accumulated in registers over the query tiles (csrc/attn_fused_bwd.cu)
            dS, dBD = _ops.attn_fused_bwd(dctx, ctx, qu, v, Pr, Pd, B, T, H, ldp, dqkv[:, d:2 * d], dqkv[:, 2 * d:],
                                          self._drop("attention_dropout"), self._seed(li, 10))
        else:
            dPd = torch.empty(H, B, T, ldt, device=dev, dtype=torch.bfloat16)
            _ops.gemm(dctx, v, dPd, T, T, hd, d, 3 * d, ldt, nb1=H, nb2=B, sA=(hd, T * d), sB=(hd, T * 3 * d),
                      sC=(B * T * ldt, T * ldt))
            # dV = Pd^T dctx
            _ops.gemm(Pd, dctx, dqkv[:, 2 * d:], T, hd, T, ldt, d, 3 * d, a_kmajor=False, b_kmajor=False, nb1=H, nb2=B,
                      sA=(B * T * ldt, T * ldt), sB=(hd, T * d), sC=(hd, T * 3 * d))
            dS, dBD = _ops.attn_softmax_bwd(Pr, dPd, T, ldp, self._drop("attention_dropout"), self._seed(li, 10))
            # dK = dS^T q_u
            _ops.gemm(dS, qu, dqkv[:, d:2 * d], T, hd, T, ldt, d, 3 * d, a_kmajor=False, b_kmajor=False, nb1=H, nb2=B,
                      sA=(B * T * ldt, T * ldt), sB=(hd, T * d), sC=(hd, T * 3 * d))
        # dq_u = dS k
        _ops.gemm(dS, k, dqu, T, hd, T, ldt, 3 * d, d, b_kmajor=False, nb1=H, nb2=B, sA=(B * T * ldt, T * ldt),
                  sB=(hd, T * 3 * d), sC=(hd, T * d))
        # dq_v = dBD P ; dP = sum_b dBD^T q_v
        learned = self.pos_tables is not None
        E = Pp.shape[1]
        ph = hd if E == d else 0
        dqv = torch.empty(R, d, device=dev, dtype=torch.bfloat16)
        # the projected positions are shared by all utterances, so the rows of all utterances form ONE M axis (B*T rows per
        # head: no partially filled 128-row tile per utterance)
        _ops.gemm(dBD, Pp, dqv, B * T, hd, 2 * T - 1, ldp, E, d, b_kmajor=False, nb1=H, nb2=1, sA=(B * T * ldp, 0),
                  sB=(ph, 0), sC=(hd, 0))
        # dpos = sum over (b, i): 2T-1 output rows per head are too few tiles to fill the machine -> split the B*T-long
        # reduction across CTAs (fp32 accumulate), then cast
        dPp32 = torch.zeros(2 * T - 1, d, device=dev, dtype=torch.float32)
        _ops.gemm(dBD, qv, dPp32, 2 * T - 1, hd, B * T, ldp, d, d, a_kmajor=False, b_kmajor=False, nb1=H, nb2=1,
                  sA=(B * T * ldp, 0), sB=(hd, 0), sC=(hd, 0), accumulate=True)
        dPp = dPp32.to(torch.bfloat16)
        _ops.qprep_bwd(dqu, dqv, self.scaling, dqkv[:, :d])
        if learned:
            # scatter-add into the table rows that were read (a width-head_dim table sums its heads first)
            _, idx = self._learned_positions(li, T, dev)
            dpe = dPp32 if E == d else dPp32.view(2 * T - 1, H, hd).sum(1)
            self.flat.grad(self.pos_tables[li]).index_add_(0, idx, dpe)
        else:
            _ops.linear_wgrad(dPp, self.pe(T, dev), self.G(lp + "self_attn.pos_proj.weight"))
            _ops.colsum(dqu, self.G(lp + "self_attn.pos_bias_u"), scale=self.scaling)
            _ops.colsum(dqv, self.G(lp + "self_attn.pos_bias_v"), scale=self.scaling)
        Wqkv, _, gW, gb = self._qkv(lp)
        _ops.linear_wgrad(dqkv, ln, gW, gb)
        dln = _ops.linear_dgrad(dqkv, Wqkv)
        return _ops.layer_norm_bwd(dln, x, mean, rstd, self.P(lp + "self_attn_layer_norm.weight"),
                                   self.G(lp + "self_attn_layer_norm.weight"), self.G(lp + "self_attn_layer_norm.bias"),
                                   dres=dy, next_drop=next_drop)

    # ---- plain scaled dot-product self-attention (absolute positions) -------------------------------
    def _plain_attn_fwd(self, q, k, v, B, T, lens, li):
        """softmax(s q k^T + key padding) v over the fused q/k/v views.  Head dim 64: the fused kernel without positions
        (q scaled first, as the learned-relative branch does); any other head dim: the unfused chain `_attend`."""
        d, H, hd = self.d, self.H, self.hd
        if self.fused_attention and hd == 64:
            if self._zeros_d is None or self._zeros_d.device != q.device:
                self._zeros_d = torch.zeros(d, device=q.device, dtype=torch.bfloat16)
            qs, _unused = _ops.qprep_fwd(q, self._zeros_d, self._zeros_d, self.scaling)
            ctx, Pr, Pd = _ops.attn_fused_fwd(qs, None, k, v, None, B, T, H, lens, self._drop("attention_dropout"),
                                              self._seed(li, 10), save_probs=self._save_probs, key_bounds=self.key_bounds)
            return ctx, ("fused", qs, Pr, Pd)
        if self.key_bounds is not None:
            raise NotImplementedError("chunk-streaming / limited-context masks run in the fused attention kernel only "
                                      "(head_dim 64, ESP_FUSED_ATTN unset)")
        ctx, att = self._attend(q, 3 * d, k, v, 3 * d, B, T, T, lens, False, li, 10)
        return ctx, ("chain",) + att

    def _plain_mha_bwd(self, dy, saved, lp, B, T, li, dyd, next_drop):
        d, H, hd = self.d, self.H, self.hd
        x, mean, rstd, ln, qkv, att, ctx = saved
        q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        dO = dyd if dyd is not None else _ops.dropout(dy, self._drop("dropout"), self._seed(li, 11))
        _ops.linear_wgrad(dO, ctx, self.G(lp + "self_attn.out_proj.weight"), self.G(lp + "self_attn.out_proj.bias"))
        dctx = _ops.linear_dgrad(dO, self.P(lp + "self_attn.out_proj.weight"))
        dqkv = torch.empty(B * T, 3 * d, device=dy.device, dtype=torch.bfloat16)
        if att[0] == "fused" and self.fused_attention_bwd:
            # dS, dK = dS^T (s q) and dV = Pd^T dctx in one kernel (no skewed copy, no frame limit); dq = s dS k
            _, qs, Pr, Pd = att
            ldt = Pr.shape[-1]
            dS, _ = _ops.attn_fused_bwd(dctx, ctx, qs, v, Pr, Pd, B, T, H, None, dqkv[:, d:2 * d], dqkv[:, 2 * d:],
                                        self._drop("attention_dropout"), self._seed(li, 10))
            _ops.gemm(dS, k, dqkv[:, :d], T, hd, T, ldt, 3 * d, 3 * d, b_kmajor=False, nb1=H, nb2=B, sA=(B * T * ldt, T * ldt),
                      sB=(hd, T * 3 * d), sC=(hd, T * 3 * d), alpha=self.scaling)
        else:
            # the unfused chain (other head dims; or ESP_FUSED_ATTN_BWD=0, from the fused forward's probabilities)
            sv = (att[2], att[3], 1.0) if att[0] == "fused" else att[1:]
            self._attend_bwd(dctx, sv, q, 3 * d, k, v, 3 * d, dqkv[:, :d], 3 * d, dqkv[:, d:2 * d], dqkv[:, 2 * d:], 3 * d,
                             B, T, T, li, 10)
        Wqkv, _, gW, gb = self._qkv(lp)
        _ops.linear_wgrad(dqkv, ln, gW, gb)
        dln = _ops.linear_dgrad(dqkv, Wqkv)
        return _ops.layer_norm_bwd(dln, x, mean, rstd, self.P(lp + "self_attn_layer_norm.weight"),
                                   self.G(lp + "self_attn_layer_norm.weight"), self.G(lp + "self_attn_layer_norm.bias"),
                                   dres=dy, next_drop=next_drop)

    # ---- unfused scaled dot-product attention (any head dim), shared with the decoder -----------------
    def _attend(self, q, ldq, k, v, ldkv, B, Tq, Tk, lens, causal, li, op, relax=0.0):
        """q [B*Tq, .] (row stride ldq), k/v [B*Tk, .] (row stride ldkv) -> ctx [B*Tq, d], saved (Pr, Pd, keep).
        relax > 0: relaxed attention (multihead_attention.py:869-872), Pd = dropout((1 - relax) P + relax / Tk); the
        backward folds keep = 1 - relax into the dq / dk GEMMs."""
        d, H, hd = self.d, self.H, self.hd
        ld = _r8(Tk)
        S = torch.empty(H, B, Tq, ld, device=q.device, dtype=torch.bfloat16)
        _ops.gemm(q, k, S, Tq, Tk, hd, ldq, ldkv, ld, nb1=H, nb2=B, sA=(hd, Tq * ldq), sB=(hd, Tk * ldkv),
                  sC=(B * Tq * ld, Tq * ld), alpha=self.scaling)
        if relax > 0:
            assert not causal
            Pr, Pd = _ops.attn_softmax_relaxed_fwd(S, Tk, lens, relax, self._drop("attention_dropout"), self._seed(li, op))
        else:
            Pr, Pd = _ops.attn_softmax_fwd(S, Tk, lens, self._drop("attention_dropout"), self._seed(li, op), causal=causal)
        ctx = torch.empty(B * Tq, d, device=q.device, dtype=torch.bfloat16)
        _ops.gemm(Pd, v, ctx, Tq, hd, Tk, ld, ldkv, d, b_kmajor=False, nb1=H, nb2=B, sA=(B * Tq * ld, Tq * ld),
                  sB=(hd, Tk * ldkv), sC=(hd, Tq * d))
        return ctx, (Pr, Pd, 1.0 - relax)

    def _attend_bwd(self, dctx, saved, q, ldq, k, v, ldkv, dq, lddq, dk, dv, lddkv, B, Tq, Tk, li, op):
        """Writes dq [B*Tq, d] (row stride lddq) and dk/dv [B*Tk, d] (row stride lddkv)."""
        d, H, hd = self.d, self.H, self.hd
        Pr, Pd, keep = saved
        ld = _r8(Tk)
        dPd = torch.empty(H, B, Tq, ld, device=dctx.device, dtype=torch.bfloat16)
        _ops.gemm(dctx, v, dPd, Tq, Tk, hd, d, ldkv, ld, nb1=H, nb2=B, sA=(hd, Tq * d), sB=(hd, Tk * ldkv),
                  sC=(B * Tq * ld, Tq * ld))
        # dV = Pd^T dctx
        _ops.gemm(Pd, dctx, dv, Tk, hd, Tq, ld, d, lddkv, a_kmajor=False, b_kmajor=False, nb1=H, nb2=B,
                  sA=(B * Tq * ld, Tq * ld), sB=(hd, Tq * d), sC=(hd, Tk * lddkv))
        # relaxed attention: with g the dropout backward of dPd, dS = keep * P (g - sum P g); the softmax backward forms
        # P (g - sum P g) and keep joins the scaling in the two GEMM alphas
        dS, _ = _ops.attn_softmax_bwd(Pr, dPd, Tk, 0, self._drop("attention_dropout"), self._seed(li, op), want_dbd=False)
        alpha = self.scaling * keep
        # dq = alpha * dS k ; dk = alpha * dS^T q
        _ops.gemm(dS, k, dq, Tq, hd, Tk, ld, ldkv, lddq, b_kmajor=False, nb1=H, nb2=B, sA=(B * Tq * ld, Tq * ld),
                  sB=(hd, Tk * ldkv), sC=(hd, Tq * lddq), alpha=alpha)
        _ops.gemm(dS, q, dk, Tk, hd, Tq, ld, ldq, lddkv, a_kmajor=False, b_kmajor=False, nb1=H, nb2=B,
                  sA=(B * Tq * ld, Tq * ld), sB=(hd, Tq * ldq), sC=(hd, Tk * lddkv), alpha=alpha)

    # ---- convolution module -----------------------------------------------------------------------
    def conv_fwd(self, x, lp, B, T, li):
        d = self.d
        cp = lp + "conv_module."
        ln, mean, rstd = _ops.layer_norm_fwd(x, self.P(cp + "layer_norm.weight"), self.P(cp + "layer_norm.bias"), LN_EPS)
        W1 = self.P(cp + "pointwise_conv1.weight").view(2 * d, d)
        Gg = _ops.linear(ln, W1)
        Wd = self.P(cp + "depthwise_conv.weight")
        ksz = Wd.shape[-1]
        Y, stats = _ops.glu_dwconv_fwd(Gg.view(B, T, 2 * d), Wd.view(d, ksz))
        rm, rv = self.bn_state[li]
        mr = _ops.bn_finalize(stats, B * T, d, BN_EPS, BN_MOMENTUM, rm, rv, self.training)
        Z = _ops.bn_silu_fwd(Y, mr, self.P(cp + "batch_norm.weight"), self.P(cp + "batch_norm.bias"))
        y = _ops.linear(Z.view(B * T, d), self.P(cp + "pointwise_conv2.weight").view(d, d), None,
                        drop_p=self._drop("dropout"), drop_mode=1, seed=self._seed(li, 20), R=x, ldr=x.stride(0), beta=1.0)
        return y, (x, mean, rstd, ln, Gg, Y, mr, Z)

    def conv_bwd(self, dy, saved, lp, B, T, li, dyd=None, next_drop=None):
        d = self.d
        cp = lp + "conv_module."
        x, mean, rstd, ln, Gg, Y, mr, Z = saved
        dO = dyd if dyd is not None else _ops.dropout(dy, self._drop("dropout"), self._seed(li, 20))
        W2 = self.P(cp + "pointwise_conv2.weight").view(d, d)
        _ops.linear_wgrad(dO, Z.view(B * T, d), self.G(cp + "pointwise_conv2.weight"))
        dZ = _ops.linear_dgrad(dO, W2)
        dY = _ops.bn_silu_bwd(dZ.view(B, T, d), Y, mr, self.P(cp + "batch_norm.weight"), self.P(cp + "batch_norm.bias"),
                              self.G(cp + "batch_norm.weight"), self.G(cp + "batch_norm.bias"))
        Wd = self.P(cp + "depthwise_conv.weight")
        ksz = Wd.shape[-1]
        dG = _ops.glu_dwconv_bwd(dY, Gg.view(B, T, 2 * d), Wd.view(d, ksz), self.G(cp + "depthwise_conv.weight").view(d, ksz))
        dG2 = dG.view(B * T, 2 * d)
        _ops.linear_wgrad(dG2, ln, self.G(cp + "pointwise_conv1.weight"))
        dln = _ops.linear_dgrad(dG2, self.P(cp + "pointwise_conv1.weight").view(2 * d, d))
        return _ops.layer_norm_bwd(dln, x, mean, rstd, self.P(cp + "layer_norm.weight"), self.G(cp + "layer_norm.weight"),
                                   self.G(cp + "layer_norm.bias"), dres=dy, next_drop=next_drop)

    # ---- layers -----------------------------------------------------------------------------------
    _CONF_FFN1 = ("ffn1.layer_norm", "ffn1.w_1", "ffn1.w_2")
    _CONF_FFN2 = ("ffn2.layer_norm", "ffn2.w_1", "ffn2.w_2")
    _TR_FFN = ("final_layer_norm", "fc1", "fc2")

    def layer_fwd(self, x, li, B, T, lens):
        lp = "layers.%d." % li
        st = {}
        if self.cfg["layer_type"] == "conformer":
            x, st["ffn1"] = self.ffn_fwd(x, lp, self._CONF_FFN1, ACT_SILU, 0.5, li, 0)
            x, st["mha"] = self.mha_fwd(x, lp, B, T, lens, li)
            x, st["conv"] = self.conv_fwd(x, lp, B, T, li)
            x, st["ffn2"] = self.ffn_fwd(x, lp, self._CONF_FFN2, ACT_SILU, 0.5, li, 2)
            y, mean, rstd = _ops.layer_norm_fwd(x, self.P(lp + "final_layer_norm.weight"), self.P(lp + "final_layer_norm.bias"), LN_EPS)
            st["final"] = (x, mean, rstd)
            return y, st
        # pre-LN Transformer block (normalize_before=True; fairseq/modules/transformer_layer.py:163-226)
        x, st["mha"] = self.mha_fwd(x, lp, B, T, lens, li)
        x, st["ffn"] = self.ffn_fwd(x, lp, self._TR_FFN, ACT_RELU, 1.0, li, 0)
        return x, st

    def layer_bwd(self, dy, st, li, B, T):
        lp = "layers.%d." % li
        if self.cfg["layer_type"] == "conformer":
            x, mean, rstd = st["final"]
            # every LayerNorm backward also writes the dropout-masked copy of its dx that the next module starts with
            pd = self._drop("dropout")
            dx, dxd = _ops.layer_norm_bwd(dy, x, mean, rstd, self.P(lp + "final_layer_norm.weight"),
                                          self.G(lp + "final_layer_norm.weight"), self.G(lp + "final_layer_norm.bias"),
                                          next_drop=(pd, self._seed(li, 3), 0.5))
            dx, dxd = self.ffn_bwd(dx, st["ffn2"], lp, self._CONF_FFN2, ACT_SILU_BWD, 0.5, li, 2, dyd=dxd,
                                   next_drop=(pd, self._seed(li, 20), 1.0))
            dx, dxd = self.conv_bwd(dx, st["conv"], lp, B, T, li, dyd=dxd, next_drop=(pd, self._seed(li, 11), 1.0))
            dx, dxd = self.mha_bwd(dx, st["mha"], lp, B, T, li, dyd=dxd, next_drop=(pd, self._seed(li, 1), 0.5))
            return self.ffn_bwd(dx, st["ffn1"], lp, self._CONF_FFN1, ACT_SILU_BWD, 0.5, li, 0, dyd=dxd)
        dx, dxd = self.ffn_bwd(dy, st["ffn"], lp, self._TR_FFN, ACT_RELU_BWD, 1.0, li, 0,
                               next_drop=(self._drop("dropout"), self._seed(li, 11), 1.0))
        return self.mha_bwd(dx, st["mha"], lp, B, T, li, dyd=dxd)

    # ---- whole encoder ----------------------------------------------------------------------------
    def forward(self, xc, lens, has_pads, save=True):
        """xc [B, T, F] bf16 (output of the conv front), lens int32 [B] (device).  Returns logits [B, T, ldV]
        (or encoder states [B, T, d] when there is no output layer) and keeps what backward needs."""
        B, T, Fin = xc.shape
        R = B * T
        cfg = self.cfg
        lens_k = lens if has_pads else None
        self._save_probs = bool(save)  # inference: the fused attention kernel writes no probabilities at all
        pdrop = self._drop("dropout")
        xin = xc.reshape(R, Fin)
        if pdrop > 0:
            xin = _ops.dropout(xin, pdrop, self._seed(999, 0))
        if self.rel_pos:
            e = _ops.linear(xin, self.P("fc0.weight"), self.P("fc0.bias"))
        else:
            # absolute positions join fc0's epilogue as its residual: one [T, d] table read by every utterance (batch
            # stride 0), e = xin W^T + b + pos (speech_transformer_encoder.py:341-345; embed_scale is 1 with fc0)
            W0 = self.P("fc0.weight")
            e = torch.empty(R, self.d, device=xc.device, dtype=torch.bfloat16)
            _ops.gemm(xin, W0, e, T, self.d, Fin, xin.stride(0), W0.stride(0), self.d, nb2=B, sA=(0, T * xin.stride(0)),
                      sC=(0, T * self.d), bias=self.P("fc0.bias"), R=self.abs_pe(T, xc.device), ldr=self.d, beta=1.0)
        if cfg.get("layernorm_embedding", False):
            x, mean0, rstd0 = _ops.layer_norm_fwd(e, self.P("layernorm_embedding.weight"), self.P("layernorm_embedding.bias"),
                                                  LN_EPS, lens=lens_k, T=T, drop_p=pdrop, seed=self._seed(999, 1))
        else:
            x = _ops.dropout(e, pdrop, self._seed(999, 1)) if pdrop > 0 else e.clone()
            if lens_k is not None:
                _ops.mask_rows_(x.view(B, T, -1), lens_k)
            mean0 = rstd0 = None
        states = []
        for li in range(cfg["layers"]):
            x, st = self.layer_fwd(x, li, B, T, lens_k)
            states.append(st)
        fin = None
        if cfg.get("final_layer_norm", False):
            xf = x
            x, mf, rf = _ops.layer_norm_fwd(xf, self.P("layer_norm.weight"), self.P("layer_norm.bias"), LN_EPS)
            fin = (xf, mf, rf)
        out = x.view(B, T, self.d)
        V = cfg.get("vocab")
        if V:
            ldV = _r8(V)
            logits = torch.zeros(R, ldV, device=x.device, dtype=torch.bfloat16) if ldV != V else \
                torch.empty(R, ldV, device=x.device, dtype=torch.bfloat16)
            _ops.gemm(x, self.P("fc_out.weight"), logits, R, V, self.d, x.stride(0), self.d, ldV, bias=self.P("fc_out.bias"))
            out = logits.view(B, T, ldV)
        if save:
            self.saved = dict(B=B, T=T, xin=xin, e=e, mean0=mean0, rstd0=rstd0, lens=lens_k, states=states, fin=fin,
                              xL=x, Fin=Fin)
        return out

    def backward(self, dout):
        """dout: gradient of the forward output ([B, T, ldV] logits or [B, T, d]).  Returns d(xc) [B, T, F]."""
        s = self.saved
        B, T = s["B"], s["T"]
        R = B * T
        cfg = self.cfg
        V = cfg.get("vocab")
        if V:
            ldV = _r8(V)
            dlog = dout.reshape(R, ldV)
            dl = dlog[:, :V] if ldV != V else dlog
            _ops.linear_wgrad(dl, s["xL"], self.G("fc_out.weight"), self.G("fc_out.bias"))
            dx = _ops.linear_dgrad(dl, self.P("fc_out.weight"))
        else:
            dx = dout.reshape(R, self.d).contiguous()
        if s["fin"] is not None:
            xf, mf, rf = s["fin"]
            dx = _ops.layer_norm_bwd(dx, xf, mf, rf, self.P("layer_norm.weight"), self.G("layer_norm.weight"),
                                     self.G("layer_norm.bias"))
        for li in reversed(range(cfg["layers"])):
            dx = self.layer_bwd(dx, s["states"][li], li, B, T)
        pdrop = self._drop("dropout")
        if cfg.get("layernorm_embedding", False):
            de = _ops.layer_norm_bwd(dx, s["e"], s["mean0"], s["rstd0"], self.P("layernorm_embedding.weight"),
                                     self.G("layernorm_embedding.weight"), self.G("layernorm_embedding.bias"),
                                     lens=s["lens"], T=T, drop_p=pdrop, seed=self._seed(999, 1))
        else:
            de = dx
            if s["lens"] is not None:
                de = _ops.mask_rows_(de.clone().view(B, T, -1), s["lens"]).view(R, -1)
            if pdrop > 0:
                de = _ops.dropout(de, pdrop, self._seed(999, 1))
        _ops.linear_wgrad(de, s["xin"], self.G("fc0.weight"), self.G("fc0.bias"))
        dxin = _ops.linear_dgrad(de, self.P("fc0.weight"))
        if pdrop > 0:
            dxin = _ops.dropout(dxin, pdrop, self._seed(999, 0))
        self.saved = None
        return dxin.view(B, T, s["Fin"])
