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

import torch

from .. import ops as _ops
from ..lib import ACT_RELU, ACT_RELU_BWD, ACT_SILU, ACT_SILU_BWD

LN_EPS = 1e-5
BN_EPS = 1e-5
BN_MOMENTUM = 0.1


def _r8(n):
    return (n + 7) // 8 * 8


def _sinusoid(lo, hi, d):
    """fp32 sinusoidal embedding of positions lo..hi-1: sin | cos halves, plus a zero column when d is odd."""
    half = d // 2
    freq = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000.0) / (half - 1)))
    pos = torch.arange(lo, hi, dtype=torch.float32)[:, None] * freq[None, :]
    emb = torch.cat([torch.sin(pos), torch.cos(pos)], dim=1)
    if d % 2 == 1:
        emb = torch.cat([emb, torch.zeros(emb.shape[0], 1)], dim=1)
    return emb


def sinusoidal_relative_table(T, d, device, dtype=torch.bfloat16):
    """Rows for relative positions -(T-1)..(T-1), scaled by d^-0.5 (scale_embedding=True), sin | cos halves.

    espresso/modules/sinusoidal_relative_positional_embedding.py:46-71,73-124 and
    espresso/modules/relative_positional_embedding.py:28-34.  Computed in fp32 then cast to the model
    dtype exactly like `self.weight.to(self._float_tensor)`."""
    return (_sinusoid(-(T - 1), T, d) * d ** -0.5).to(device=device, dtype=dtype).contiguous()


def sinusoidal_positions(U, d, padding_idx, device, dtype=torch.bfloat16):
    """Rows t = 0..U-1 of fairseq's sinusoidal table at index t + padding_idx + 1 (right-padded sequences),
    computed in fp32 then cast to the model dtype."""
    return _sinusoid(padding_idx + 1, padding_idx + 1 + U, d).to(device=device, dtype=dtype).contiguous()


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
        self._save_probs = True
        self.key_bounds = None  # (lo, hi) int32 [T] device tensors: per-row visible key range (streaming masks)

    # ------------------------------------------------------------------------------------------
    def P(self, name):
        return self.flat.param(self.pre + name)

    def G(self, name):
        return self.flat.grad(self.pre + name)

    def _proj(self, lp, which, names):
        """The adjacent projections `which`.{names}_proj of layer prefix lp as one stacked Linear:
        (weight bf16, bias bf16, weight grad fp32, bias grad fp32), views of the flat buffers."""
        ws = [self.pre + lp + "%s.%s_proj.weight" % (which, c) for c in names]
        bs = [self.pre + lp + "%s.%s_proj.bias" % (which, c) for c in names]
        n, d = len(names), self.d
        return (self.flat.span(self.flat.p16, ws, (n * d, d)), self.flat.span(self.flat.p16, bs, (n * d,)),
                self.flat.span(self.flat.g32, ws, (n * d, d)), self.flat.span(self.flat.g32, bs, (n * d,)))

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

    # ---- multi-head self-attention -----------------------------------------------------------------
    def _scaled_q(self, q):
        """q * scaling as qprep_fwd forms it with zero biases, contiguous."""
        if self._zeros_d is None or self._zeros_d.device != q.device:
            self._zeros_d = torch.zeros(self.d, device=q.device, dtype=torch.bfloat16)
        return _ops.qprep_fwd(q, self._zeros_d, self._zeros_d, self.scaling)[0]

    def mha_fwd(self, x, lp, B, T, lens, li):
        """x + dropout(out_proj(self-attention(LayerNorm(x)))).  The position source only changes how q is prepared and
        whether relative-position logits join the scores: sinusoidal rows through pos_proj with pos_bias_u / pos_bias_v,
        learned table rows, or none (absolute positions were added after fc0).  Head dim 64 runs the fused kernels
        (csrc/attn_fused.cu, csrc/attn_fused_bwd.cu), any other the unfused chain `_attend`."""
        d, hd = self.d, self.hd
        ln, mean, rstd = _ops.layer_norm_fwd(x, self.P(lp + "self_attn_layer_norm.weight"),
                                             self.P(lp + "self_attn_layer_norm.bias"), LN_EPS)
        Wqkv, bqkv, _, _ = self._proj(lp, "self_attn", "qkv")
        qkv = _ops.linear(ln, Wqkv, bqkv)
        q, k, v = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
        fused = hd == 64
        pos = None  # relative positions: (q_v, rows P [2T-1, E], head stride of P)
        if not self.rel_pos:
            # the fused kernel takes q scaled first; the unfused chain scales in its score GEMM
            qu = self._scaled_q(q) if fused else q
        else:
            if self.pos_tables is None:
                qu, qv = _ops.qprep_fwd(q, self.P(lp + "self_attn.pos_bias_u"), self.P(lp + "self_attn.pos_bias_v"),
                                        self.scaling)
                Pp = _ops.linear(self.pe(T, x.device), self.P(lp + "self_attn.pos_proj.weight"))  # batch independent
            else:
                # learned tables: q is only scaled (no pos_bias_u / pos_bias_v), the rows are used as they are (no pos_proj)
                qu = qv = self._scaled_q(q)
                Pp, _ = self._learned_positions(li, T, x.device)
            pos = (qv, Pp, hd if Pp.shape[1] == d else 0)  # a table of width head_dim serves all heads (head stride 0)
        # alpha of the q-side gradient GEMMs: q_u is already scaled (qprep_bwd applies the scaling), q is not
        scale = 1.0 if pos is not None else self.scaling
        if fused:
            # scores, position logits and skew, masks, softmax and P v in ONE kernel; only the probabilities the backward
            # needs go to HBM
            qv, Pp, ph = pos or (None, None, None)
            ctx, Pr, Pd = _ops.attn_fused_fwd(qu, qv, k, v, Pp, B, T, self.H, lens, self._drop("attention_dropout"),
                                              self._seed(li, 10), save_probs=self._save_probs, pos_hstride=ph,
                                              key_bounds=self.key_bounds)
            att = (Pr, Pd, scale)
        else:
            if self.key_bounds is not None:
                raise NotImplementedError("chunk-streaming / limited-context masks run in the fused attention kernel only, "
                                          "which needs head_dim 64 (this model has head_dim %d)" % hd)
            ctx, att = self._attend(qu, qu.stride(0), k, v, 3 * d, B, T, T, lens, False, li, 10, scale=scale, pos=pos)
        y = _ops.linear(ctx, self.P(lp + "self_attn.out_proj.weight"), self.P(lp + "self_attn.out_proj.bias"),
                        drop_p=self._drop("dropout"), drop_mode=1, seed=self._seed(li, 11), R=x, ldr=x.stride(0), beta=1.0)
        # the fused backward's skew kernel takes rows of at most 1024 keys; without positions it does not run
        fused_bwd = fused and (pos is None or T <= 1024)
        return y, (x, mean, rstd, ln, qkv, qu, pos, att, ctx, fused_bwd)

    def mha_bwd(self, dy, saved, lp, B, T, li, dyd=None, next_drop=None):
        d, H, hd = self.d, self.H, self.hd
        R = B * T
        x, mean, rstd, ln, qkv, qu, pos, att, ctx, fused_bwd = saved
        k, v = qkv[:, d:2 * d], qkv[:, 2 * d:]
        dev = dy.device
        dO = dyd if dyd is not None else _ops.dropout(dy, self._drop("dropout"), self._seed(li, 11))
        _ops.linear_wgrad(dO, ctx, self.G(lp + "self_attn.out_proj.weight"), self.G(lp + "self_attn.out_proj.bias"))
        dctx = _ops.linear_dgrad(dO, self.P(lp + "self_attn.out_proj.weight"))
        dqkv = torch.empty(R, 3 * d, device=dev, dtype=torch.bfloat16)
        # with relative positions the score side yields d(q_u); qprep_bwd below turns it and d(q_v) into dq
        dq = torch.empty(R, d, device=dev, dtype=torch.bfloat16) if pos is not None else dqkv[:, :d]
        ldp = _r8(2 * T - 1) if pos is not None else None
        if fused_bwd:
            # ONE kernel: dPd = dctx v^T and dS in registers (dS written once, plus its skewed copy dBD with positions),
            # dV = Pd^T dctx and dK = dS^T q_u accumulated over the query tiles; then dq = alpha dS k
            Pr, Pd, alpha = att
            dS, dBD = _ops.attn_fused_bwd(dctx, ctx, qu, v, Pr, Pd, B, T, H, ldp, dqkv[:, d:2 * d], dqkv[:, 2 * d:],
                                          self._drop("attention_dropout"), self._seed(li, 10))
            ldt = _r8(T)
            _ops.gemm(dS, k, dq, T, hd, T, ldt, 3 * d, dq.stride(0), b_kmajor=False, nb1=H, nb2=B,
                      sA=(B * T * ldt, T * ldt), sB=(hd, T * 3 * d), sC=(hd, T * dq.stride(0)), alpha=alpha)
        else:
            dBD = self._attend_bwd(dctx, att, qu, qu.stride(0), k, v, 3 * d, dq, dq.stride(0), dqkv[:, d:2 * d],
                                   dqkv[:, 2 * d:], 3 * d, B, T, T, li, 10, ldp=ldp)
        if pos is not None:
            qv, Pp, ph = pos
            E = Pp.shape[1]
            # dq_v = dBD P ; dP = sum_b dBD^T q_v.  The positions are shared by all utterances, so the rows of all
            # utterances form ONE M axis (B*T rows per head: no partially filled 128-row tile per utterance)
            dqv = torch.empty(R, d, device=dev, dtype=torch.bfloat16)
            _ops.gemm(dBD, Pp, dqv, B * T, hd, 2 * T - 1, ldp, E, d, b_kmajor=False, nb1=H, nb2=1, sA=(B * T * ldp, 0),
                      sB=(ph, 0), sC=(hd, 0))
            # dpos = sum over (b, i): 2T-1 output rows per head are too few tiles to fill the machine -> split the
            # B*T-long reduction across CTAs (fp32 accumulate), then cast
            dPp32 = torch.zeros(2 * T - 1, d, device=dev, dtype=torch.float32)
            _ops.gemm(dBD, qv, dPp32, 2 * T - 1, hd, B * T, ldp, d, d, a_kmajor=False, b_kmajor=False, nb1=H, nb2=1,
                      sA=(B * T * ldp, 0), sB=(hd, 0), sC=(hd, 0), accumulate=True)
            dPp = dPp32.to(torch.bfloat16)
            _ops.qprep_bwd(dq, dqv, self.scaling, dqkv[:, :d])
            if self.pos_tables is not None:
                # scatter-add into the table rows that were read (a width-head_dim table sums its heads first)
                _, idx = self._learned_positions(li, T, dev)
                dpe = dPp32 if E == d else dPp32.view(2 * T - 1, H, hd).sum(1)
                self.flat.grad(self.pos_tables[li]).index_add_(0, idx, dpe)
            else:
                _ops.linear_wgrad(dPp, self.pe(T, dev), self.G(lp + "self_attn.pos_proj.weight"))
                _ops.colsum(dq, self.G(lp + "self_attn.pos_bias_u"), scale=self.scaling)
                _ops.colsum(dqv, self.G(lp + "self_attn.pos_bias_v"), scale=self.scaling)
        Wqkv, _, gW, gb = self._proj(lp, "self_attn", "qkv")
        _ops.linear_wgrad(dqkv, ln, gW, gb)
        dln = _ops.linear_dgrad(dqkv, Wqkv)
        return _ops.layer_norm_bwd(dln, x, mean, rstd, self.P(lp + "self_attn_layer_norm.weight"),
                                   self.G(lp + "self_attn_layer_norm.weight"), self.G(lp + "self_attn_layer_norm.bias"),
                                   dres=dy, next_drop=next_drop)

    # ---- unfused scaled dot-product attention (any head dim), shared with the decoder -----------------
    def _attend(self, q, ldq, k, v, ldkv, B, Tq, Tk, lens, causal, li, op, relax=0.0, scale=None, pos=None):
        """q [B*Tq, .] (row stride ldq), k/v [B*Tk, .] (row stride ldkv) -> ctx [B*Tq, d], saved (Pr, Pd, alpha).
        scale: alpha of the score GEMM, head_dim^-0.5 when None (q unscaled); 1 for a q scaled beforehand.
        pos: relative positions (q_v [B*Tq, d], rows P [2Tk-1, E], head stride of P): the BD GEMM forms q_v P^T and the
        score GEMM adds it in skewed layout.
        relax > 0: relaxed attention (multihead_attention.py:869-872), Pd = dropout((1 - relax) P + relax / Tk).
        alpha = scale * (1 - relax) is what the backward's dq / dk GEMMs take."""
        d, H, hd = self.d, self.H, self.hd
        scale = self.scaling if scale is None else scale
        rel = {}
        if pos is not None:
            qv, Pp, ph = pos
            ldp = _r8(2 * Tk - 1)
            BD = torch.empty(H, B, Tq, ldp, device=q.device, dtype=torch.bfloat16)
            _ops.gemm(qv, Pp, BD, Tq, 2 * Tk - 1, hd, qv.stride(0), Pp.shape[1], ldp, nb1=H, nb2=B,
                      sA=(hd, Tq * qv.stride(0)), sB=(ph, 0), sC=(B * Tq * ldp, Tq * ldp))
            rel = dict(R=BD, ldr=ldp, sR=(B * Tq * ldp, Tq * ldp), skew_r=Tk)
        ld = _r8(Tk)
        S = torch.empty(H, B, Tq, ld, device=q.device, dtype=torch.bfloat16)
        _ops.gemm(q, k, S, Tq, Tk, hd, ldq, ldkv, ld, nb1=H, nb2=B, sA=(hd, Tq * ldq), sB=(hd, Tk * ldkv),
                  sC=(B * Tq * ld, Tq * ld), alpha=scale, **rel)
        if relax > 0:
            assert not causal
            Pr, Pd = _ops.attn_softmax_relaxed_fwd(S, Tk, lens, relax, self._drop("attention_dropout"), self._seed(li, op))
        else:
            Pr, Pd = _ops.attn_softmax_fwd(S, Tk, lens, self._drop("attention_dropout"), self._seed(li, op), causal=causal)
        ctx = torch.empty(B * Tq, d, device=q.device, dtype=torch.bfloat16)
        _ops.gemm(Pd, v, ctx, Tq, hd, Tk, ld, ldkv, d, b_kmajor=False, nb1=H, nb2=B, sA=(B * Tq * ld, Tq * ld),
                  sB=(hd, Tk * ldkv), sC=(hd, Tq * d))
        return ctx, (Pr, Pd, scale * (1.0 - relax))

    def _attend_bwd(self, dctx, saved, q, ldq, k, v, ldkv, dq, lddq, dk, dv, lddkv, B, Tq, Tk, li, op, ldp=None):
        """Writes dq [B*Tq, d] (row stride lddq) and dk/dv [B*Tk, d] (row stride lddkv).  ldp: the forward had relative
        positions; returns dBD [H, B, Tq, ldp], the score gradient in their skewed layout (None without)."""
        d, H, hd = self.d, self.H, self.hd
        Pr, Pd, alpha = saved
        ld = _r8(Tk)
        dPd = torch.empty(H, B, Tq, ld, device=dctx.device, dtype=torch.bfloat16)
        _ops.gemm(dctx, v, dPd, Tq, Tk, hd, d, ldkv, ld, nb1=H, nb2=B, sA=(hd, Tq * d), sB=(hd, Tk * ldkv),
                  sC=(B * Tq * ld, Tq * ld))
        # dV = Pd^T dctx
        _ops.gemm(Pd, dctx, dv, Tk, hd, Tq, ld, d, lddkv, a_kmajor=False, b_kmajor=False, nb1=H, nb2=B,
                  sA=(B * Tq * ld, Tq * ld), sB=(hd, Tq * d), sC=(hd, Tk * lddkv))
        # relaxed attention: with g the dropout backward of dPd, dS = keep * P (g - sum P g), keep = 1 - relax; the
        # softmax backward forms P (g - sum P g) and keep is part of alpha
        dS, dBD = _ops.attn_softmax_bwd(Pr, dPd, Tk, ldp or 0, self._drop("attention_dropout"), self._seed(li, op),
                                        want_dbd=ldp is not None)
        # dq = alpha * dS k ; dk = alpha * dS^T q
        _ops.gemm(dS, k, dq, Tq, hd, Tk, ld, ldkv, lddq, b_kmajor=False, nb1=H, nb2=B, sA=(B * Tq * ld, Tq * ld),
                  sB=(hd, Tk * ldkv), sC=(hd, Tq * lddq), alpha=alpha)
        _ops.gemm(dS, q, dk, Tk, hd, Tq, ld, ldq, lddkv, a_kmajor=False, b_kmajor=False, nb1=H, nb2=B,
                  sA=(B * Tq * ld, Tq * ld), sB=(hd, Tq * ldq), sC=(hd, Tk * lddkv), alpha=alpha)
        return dBD

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
