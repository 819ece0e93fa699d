"""`speech_transformer_encoder_model` (CTC / encoder-only Transformer or Conformer), H100-native.

Mirrors the reference's public surface so criterions/decoders written for it keep working:
  espresso/models/transformer/speech_transformer_encoder_model.py:35-210
      SpeechTransformerEncoderModel.build_model / forward / get_normalized_probs / output_lengths
      SpeechTransformerEncoderForPrediction (encoder + fc_out)
  espresso/models/transformer/speech_transformer_encoder.py:48-409  (SpeechTransformerEncoderBase)
  espresso/modules/speech_convolutions.py:20-102                      (ConvBNReLU)
Parameter names (state_dict keys) are identical to the reference's, so checkpoints interchange.
The modules below are *containers*: they own parameters (re-homed into one flat bf16 buffer by
`finalize_()`), while the arithmetic runs in `EncoderEngine` over libespresso_b200.so.
"""
import math

import numpy as np

import torch
import torch.nn as nn
import torch.nn.functional as F

from ... import ops as _ops
from ...flat import FlatParams
from ...modules.encoder_engine import EncoderEngine
from ...data.specaugment import numpy_seed
from ...registry import register_model
from ...tools.utils import chunk_streaming_bounds, context_bounds
from .speech_transformer_config import DEFAULT_MAX_SOURCE_POSITIONS, SpeechTransformerConfig, eval_str_nested_list_or_tuple


# ---------------------------------------------------------------------------------------------------
# parameter containers (names == reference)
# ---------------------------------------------------------------------------------------------------
def _xavier(t, gain=1.0):
    nn.init.xavier_uniform_(t, gain=gain)
    return t


class _Affine(nn.Module):  # LayerNorm container
    def __init__(self, d):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d))
        self.bias = nn.Parameter(torch.zeros(d))


class _Linear(nn.Module):
    def __init__(self, i, o, bias=True, xavier=None):
        super().__init__()
        lin = nn.Linear(i, o, bias=bias)  # default torch init (fairseq/modules/conformer_layer.py:128-129)
        if xavier is not None:            # fairseq Linear helper / MHA init (multihead_attention.py:190-212)
            _xavier(lin.weight, xavier)
            if bias:
                nn.init.constant_(lin.bias, 0.0)
        self.weight = lin.weight
        if bias:
            self.bias = lin.bias


class _PosEmbStub(nn.Module):
    """Keeps the `_float_tensor` buffer key of the reference's sinusoidal position modules (a relative-position layer's
    `positional_embedding`, the absolute-position encoder's `embed_positions`)."""
    def __init__(self):
        super().__init__()
        self.register_buffer("_float_tensor", torch.zeros(1))


class _LearnedRelPos(nn.Module):
    """espresso/modules/learned_relative_positional_embedding.py:13-45: table of 2*max_size-1 relative positions
    (padding_idx None), N(0, dim^-0.5) init; state_dict key `weight` like the reference's nn.Embedding."""
    def __init__(self, dim, max_size):
        super().__init__()
        self.max_size = max_size
        self.weight = nn.Parameter(torch.empty(2 * max_size - 1, dim))
        nn.init.normal_(self.weight, mean=0.0, std=dim ** -0.5)


class _SelfAttn(nn.Module):
    def __init__(self, d, H, positional_embedding=None, relative=True):
        """positional_embedding: None -> sinusoidal relative positions (pos_bias_u/v + pos_proj, Transformer-XL);
        a _LearnedRelPos -> learned table, no biases / projection (fairseq/modules/multihead_attention.py:150-167).
        relative=False: plain scaled dot-product attention, no position parameters at all (:166)."""
        super().__init__()
        g = 1 / math.sqrt(2)
        if positional_embedding is None and relative:
            self.pos_bias_u = nn.Parameter(torch.empty(d))
            self.pos_bias_v = nn.Parameter(torch.empty(d))
            nn.init.xavier_uniform_(self.pos_bias_u.data.view(H, -1))
            nn.init.xavier_uniform_(self.pos_bias_v.data.view(H, -1))
        self.k_proj = _Linear(d, d, xavier=g)
        self.v_proj = _Linear(d, d, xavier=g)
        self.q_proj = _Linear(d, d, xavier=g)
        self.out_proj = _Linear(d, d, xavier=1.0)
        if relative and positional_embedding is None:
            self.positional_embedding = _PosEmbStub()
            self.pos_proj = _Linear(d, d, bias=False, xavier=g)
        elif relative:
            self.positional_embedding = positional_embedding


class _FFN(nn.Module):
    def __init__(self, d, ffn):
        super().__init__()
        self.layer_norm = _Affine(d)
        self.w_1 = _Linear(d, ffn)
        self.w_2 = _Linear(ffn, d)


class _BN(nn.Module):
    def __init__(self, c):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(c))
        self.bias = nn.Parameter(torch.zeros(c))
        self.register_buffer("running_mean", torch.zeros(c))
        self.register_buffer("running_var", torch.ones(c))
        self.register_buffer("num_batches_tracked", torch.tensor(0, dtype=torch.long))

    def fp32_running_stats_(self):
        """The native BatchNorm kernels read and update fp32 running statistics, whatever the parameters' dtype."""
        self.running_mean.data = self.running_mean.data.float()
        self.running_var.data = self.running_var.data.float()


class _ConvModule(nn.Module):
    def __init__(self, d, k):
        super().__init__()
        self.layer_norm = _Affine(d)
        self.pointwise_conv1 = nn.Conv1d(d, 2 * d, 1, bias=False)
        self.depthwise_conv = nn.Conv1d(d, d, k, padding=(k - 1) // 2, groups=d, bias=False)
        self.batch_norm = _BN(d)
        self.pointwise_conv2 = nn.Conv1d(d, d, 1, bias=False)


class _ConformerLayer(nn.Module):
    def __init__(self, d, ffn, H, k, positional_embedding=None, relative=True):
        super().__init__()
        self.ffn1 = _FFN(d, ffn)
        self.self_attn = _SelfAttn(d, H, positional_embedding, relative)
        self.self_attn_layer_norm = _Affine(d)
        self.conv_module = _ConvModule(d, k)
        self.ffn2 = _FFN(d, ffn)
        self.final_layer_norm = _Affine(d)


class _TransformerLayer(nn.Module):
    def __init__(self, d, ffn, H, positional_embedding=None, relative=True):
        super().__init__()
        self.self_attn = _SelfAttn(d, H, positional_embedding, relative)
        self.self_attn_layer_norm = _Affine(d)
        self.fc1 = _Linear(d, ffn, xavier=1.0)
        self.fc2 = _Linear(ffn, d, xavier=1.0)
        self.final_layer_norm = _Affine(d)


class _BNReLUFn(torch.autograd.Function):
    """BatchNorm2d (batch statistics) + ReLU on a channels-last activation, forward and backward in the native
    kernels (esp_bn_stats / esp_bn_finalize / esp_bn_act_fwd / esp_bn_act_bwd).  x is [B, C, T, F] with
    channels_last strides, i.e. memory [B, T, F, C]."""

    @staticmethod
    def forward(ctx, x, bn, gw, gb, training, conv_bias):
        xr = x.permute(0, 2, 3, 1)  # [B, T, F, C] contiguous view
        assert xr.is_contiguous()
        C = xr.shape[-1]
        R = xr.numel() // C
        stats = _ops.bn_stats(xr, C, pre_bias=conv_bias) if training else None
        mr = _ops.bn_finalize(stats, R, C, 1e-5, 0.1, bn.running_mean, bn.running_var, training)
        z = _ops.bn_act_fwd(xr, mr, bn.weight.data, bn.bias.data, _ops.BN_ACT_RELU, pre_bias=conv_bias)
        ctx.save_for_backward(xr, mr)
        ctx.bn, ctx.gw, ctx.gb, ctx.conv_bias = bn, gw, gb, conv_bias
        return z.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, dz):
        xr, mr = ctx.saved_tensors
        dzr = dz.permute(0, 2, 3, 1).contiguous()
        dx = _ops.bn_act_bwd(dzr, xr, mr, ctx.bn.weight.data, ctx.bn.bias.data, ctx.gw, ctx.gb, _ops.BN_ACT_RELU,
                             pre_bias=ctx.conv_bias)
        return dx.permute(0, 3, 1, 2), None, None, None, None, None


class _ConvBNReLUFn(torch.autograd.Function):
    """One conv-front layer on channels-last rows [B, T, F, C]: native 3x3 convolution (esp_conv3x3_*: implicit GEMM on the
    wgmma kernel, or the direct kernel of the one-channel first layer) -> BatchNorm2d (batch statistics) -> ReLU.
    The convolution weight and BatchNorm parameter gradients are accumulated straight into the flat fp32 buffer
    (`gw`, `gbw`, `gbb`); the convolution bias sits inside the BatchNorm kernels (`conv_bias`, see ConvBNReLU.forward).
    `anchor` only makes autograd call backward when the features themselves need no gradient (first layer)."""

    @staticmethod
    def forward(ctx, x, anchor, w, gw, stride, bn, gbw, gbb, training, conv_bias, need_dx):
        y = _ops.conv3x3_fwd(x, w, stride)
        C = y.shape[-1]
        R = y.numel() // C
        stats = _ops.bn_stats(y, C, pre_bias=conv_bias) if training else None
        mr = _ops.bn_finalize(stats, R, C, 1e-5, 0.1, bn.running_mean, bn.running_var, training)
        z = _ops.bn_act_fwd(y, mr, bn.weight.data, bn.bias.data, _ops.BN_ACT_RELU, pre_bias=conv_bias)
        ctx.save_for_backward(x, y, mr)
        ctx.w, ctx.gw, ctx.stride, ctx.bn, ctx.gbw, ctx.gbb, ctx.conv_bias, ctx.need_dx = w, gw, stride, bn, gbw, gbb, conv_bias, need_dx
        return z

    @staticmethod
    def backward(ctx, dz):
        x, y, mr = ctx.saved_tensors
        dy = _ops.bn_act_bwd(dz.contiguous(), y, mr, ctx.bn.weight.data, ctx.bn.bias.data, ctx.gbw, ctx.gbb, _ops.BN_ACT_RELU,
                             pre_bias=ctx.conv_bias)
        _ops.conv3x3_wgrad(dy, x, ctx.gw, ctx.stride)
        dx = _ops.conv3x3_dgrad(dy, ctx.w, tuple(x.shape), ctx.stride) if ctx.need_dx else None
        return (dx,) + (None,) * 10


class ConvBNReLU(nn.Module):
    """espresso/modules/speech_convolutions.py:20-102.  (Conv2d 3x3 -> BatchNorm2d -> ReLU) x N, then
    [B, C, T', F'] -> [B, T', C*F'].  Activations and conv weights are kept channels-last ([B, T, F, C] rows, weights
    [Cout, 3, 3, Cin] in the flat buffers); every layer runs in the native kernels: the 3x3 convolutions and their input /
    weight gradients as implicit GEMMs on the wgmma kernel (csrc/gemm_tcgen05.cu ConvGeom: im2col tiles are TMA boxes of
    the activation shifted by the filter tap), the one-input-channel first layer as a direct kernel, BatchNorm + ReLU
    (forward, backward, running statistics) in the row kernels.  Layer shapes outside the native kernels' domain (kernel
    other than 3x3, stride > 2, channel counts that are not multiples of 64) fall back to the library convolution.
    The reference's zeroing of padded frames at this point (:97-100) is dropped: the encoder zeroes the same rows again
    after fc0 / layernorm_embedding (speech_transformer_encoder.py:354-357), which makes the first one a no-op."""

    def __init__(self, out_channels, kernel_sizes, strides, in_channels=1):
        super().__init__()
        self.out_channels, self.kernel_sizes, self.strides, self.in_channels = out_channels, kernel_sizes, strides, in_channels
        self.convolutions = nn.ModuleList()
        self.batchnorms = nn.ModuleList()
        cin = in_channels
        for c, k, s in zip(out_channels, kernel_sizes, strides):
            k = tuple(k) if isinstance(k, (list, tuple)) else (k, k)
            s = tuple(s) if isinstance(s, (list, tuple)) else (s, s)
            self.convolutions.append(nn.Conv2d(cin, c, k, stride=s, padding=((k[0] - 1) // 2, (k[1] - 1) // 2)))
            self.batchnorms.append(_BN(c))
            cin = c
        self.flat = None
        self.flat_prefix = ""
        self._anchor = None

    @classmethod
    def from_config(cls, conv_channels, conv_kernel_sizes, conv_strides, feat_dim, in_channels):
        """The conv front of the config strings (the reference's encoder_conv_* / encoder.conv_* options) over features of
        `feat_dim` = in_channels x frequency bins.  Returns (front, its output width), or (None, feat_dim) without one."""
        out_channels = eval_str_nested_list_or_tuple(conv_channels)
        if out_channels is None:
            return None, feat_dim
        assert feat_dim % in_channels == 0
        front = cls(out_channels, eval_str_nested_list_or_tuple(conv_kernel_sizes),
                    eval_str_nested_list_or_tuple(conv_strides), in_channels=in_channels)
        return front, front.output_width(feat_dim)

    def output_lengths(self, in_lengths):
        out = in_lengths
        for s in self.strides:
            s0 = s[0] if isinstance(s, (list, tuple)) else s
            out = torch.div(out + s0 - 1, s0, rounding_mode="floor") if torch.is_tensor(out) else (out + s0 - 1) // s0
        return out

    def output_width(self, feat_dim):
        """Width of [B, T', C * F'] after the front: the frequency axis is subsampled by the second stride of each layer."""
        size = feat_dim // self.in_channels
        for s in self.strides:
            s1 = (s[1] if len(s) > 1 else s[0]) if isinstance(s, (list, tuple)) else s
            size = (size + s1 - 1) // s1
        return size * self.out_channels[-1]

    def channels_last_weights(self, prefix):
        """Flat names of the convolution weights, which the flat buffers store [Cout, kh, kw, Cin] (see forward)."""
        return [prefix + "convolutions.%d.weight" % i for i in range(len(self.convolutions))]

    def use_flat_(self, flat, prefix):
        """Run on the flat buffers' views and gradients of this front's parameters, named prefix + local name."""
        self.flat, self.flat_prefix = flat, prefix
        for bn in self.batchnorms:
            bn.fp32_running_stats_()

    def native_convolutions(self):
        """True when every layer is inside the native kernels' domain (all shipped recipes: 3x3, strides 1 / 2,
        1 -> 64 -> 64 -> 128 -> 128 channels)."""
        cin = self.in_channels
        for conv in self.convolutions:
            c = conv.out_channels
            if tuple(conv.kernel_size) != (3, 3) or any(s not in (1, 2) for s in conv.stride):
                return False
            if cin == 1:
                if c % 8 or c > 256 or 256 % (c // 8):
                    return False
            elif cin % 64 or c % 64:
                return False
            cin = c
        return True

    def forward(self, src, src_lengths):
        if not self.native_convolutions():
            return self._forward_library(src, src_lengths)
        B, T, D = src.shape
        cin = self.in_channels
        # [B, T, cin * F] (channel-major feature axis, :80-86) -> channels-last rows [B, T, F, cin]; one channel: [B, T, F]
        x = src.contiguous() if cin == 1 else src.view(B, T, cin, D // cin).transpose(2, 3).contiguous()
        if self._anchor is None or self._anchor.device != src.device:
            self._anchor = torch.zeros(1, device=src.device, requires_grad=True)
        for i, (conv, bn) in enumerate(zip(self.convolutions, self.batchnorms)):
            name = self.flat_prefix + "convolutions.%d.weight" % i
            w = self.flat.param(name).permute(0, 2, 3, 1)   # the flat storage order: [Cout, 3, 3, Cin], contiguous
            gw = self.flat.grad(name).permute(0, 2, 3, 1)
            gbw = self.flat.grad(self.flat_prefix + "batchnorms.%d.weight" % i)
            gbb = self.flat.grad(self.flat_prefix + "batchnorms.%d.bias" % i)
            if self.training:
                bn.num_batches_tracked += 1
            # The convolution runs WITHOUT its bias: the bias is added inside the BatchNorm kernels (pre_bias), which
            # removes one full pass over the activation in forward (bias add) and one in backward (bias-gradient
            # reduction).  The gradient of a bias in front of a batch-statistics BatchNorm is identically zero
            # (the reference computes rounding noise there), so conv.bias receives no gradient.
            x = _ConvBNReLUFn.apply(x, self._anchor, w, gw, tuple(conv.stride), bn, gbw, gbb, self.training,
                                    conv.bias.data if conv.bias is not None else None, i > 0 or src.requires_grad)
        # [B, T', F', C] -> [B, T', C * F']   (channel-major inner index, as in the reference :92-94)
        x = x.transpose(2, 3).reshape(x.size(0), x.size(1), x.size(2) * x.size(3))
        return x, self.output_lengths(src_lengths)

    def _forward_library(self, src, src_lengths):
        x = src.view(src.size(0), src.size(1), self.in_channels, src.size(2) // self.in_channels).transpose(1, 2)
        x = x.contiguous(memory_format=torch.channels_last)
        for i, (conv, bn) in enumerate(zip(self.convolutions, self.batchnorms)):
            x = F.conv2d(x, conv.weight, None, conv.stride, conv.padding)
            if not x.is_contiguous(memory_format=torch.channels_last):
                x = x.contiguous(memory_format=torch.channels_last)
            gw = self.flat.grad(self.flat_prefix + "batchnorms.%d.weight" % i)
            gb = self.flat.grad(self.flat_prefix + "batchnorms.%d.bias" % i)
            if self.training:
                bn.num_batches_tracked += 1
            x = _BNReLUFn.apply(x, bn, gw, gb, self.training, conv.bias.data if conv.bias is not None else None)
        # B x C x T' x F' -> B x T' x (C * F')   (channel-major inner index, as in the reference)
        x = x.permute(0, 2, 1, 3).contiguous()
        x = x.view(x.size(0), x.size(1), x.size(2) * x.size(3))
        return x, self.output_lengths(src_lengths)


class _EncoderFn(torch.autograd.Function):
    """One autograd node for the whole encoder stack: forward/backward are the hand-written engine passes;
    parameter gradients go straight into the flat fp32 buffer (nothing is returned for them)."""

    @staticmethod
    def forward(ctx, xc, anchor, engine, lens, has_pads):
        ctx.engine = engine
        return engine.forward(xc, lens, has_pads, save=torch.is_grad_enabled() or True)

    @staticmethod
    def backward(ctx, dout):
        dxc = ctx.engine.backward(dout.contiguous())
        # a host that drives plain autograd (fairseq's trainer through espresso_b200_plugin) asks to be called once the
        # WHOLE backward pass is over, to publish the flat fp32 gradients as .grad
        cb = getattr(ctx.engine, "after_backward", None)
        if cb is not None:
            torch.autograd.Variable._execution_engine.queue_callback(cb)
        return dxc, None, None, None, None


class SpeechTransformerEncoderForPrediction(nn.Module):
    """Encoder (+ optional fc_out).  forward returns the reference's dict of lists
    (speech_transformer_encoder.py:399-409) with `encoder_out` = T' x B x V."""

    def __init__(self, cfg: SpeechTransformerConfig, pre_encoder=None, input_size=83, vocab_size=None):
        super().__init__()
        self.cfg = cfg
        e = cfg.encoder
        rel = e.relative_positional_embeddings
        if not rel and e.learned_pos:
            raise NotImplementedError("native encoder: learned absolute positional embeddings are not supported (no recipe "
                                      "uses them); use sinusoidal absolute (learned_pos=False) or relative positions")
        if not rel and cfg.no_token_positional_embeddings:
            raise NotImplementedError("native encoder: an encoder without any positional embeddings is not supported")
        if not e.normalize_before:
            raise NotImplementedError("post-LN encoder layers are not on the recipes' path")
        self.register_buffer("version", torch.Tensor([3]))
        self.pre_encoder = pre_encoder
        d = e.embed_dim
        self.max_source_positions = cfg.max_source_positions
        self.fc0 = _Linear(input_size, d, xavier=1.0)
        # absolute positions (relative_positional_embeddings off: the WSJ / Switchboard Transformer recipes): fairseq's
        # sinusoidal table, added after fc0 (speech_transformer_encoder.py:93-101,343-345); no parameters, one buffer key
        if not rel:
            self.embed_positions = _PosEmbStub()
        self.layernorm_embedding = _Affine(d) if cfg.layernorm_embedding else None
        # relative position source per layer (speech_transformer_encoder.py:121-158): sinusoidal (None here), or
        # learned tables -- per layer or one shared instance, of width d or head_dim (shared across heads)
        if rel and e.learned_pos:
            max_size = int(self.output_lengths(cfg.max_source_positions)) if pre_encoder is not None else cfg.max_source_positions
            dim = d // e.attention_heads if e.share_learned_relative_positional_embeddings_across_heads else d
            if e.share_learned_relative_positional_embeddings_across_layers:
                pos = [_LearnedRelPos(dim, max_size)] * e.layers
            else:
                pos = [_LearnedRelPos(dim, max_size) for _ in range(e.layers)]
        else:
            pos = [None] * e.layers
        if e.layer_type == "conformer":
            self.layers = nn.ModuleList([_ConformerLayer(d, e.ffn_embed_dim, e.attention_heads, e.depthwise_conv_kernel_size,
                                                         pos[i], rel) for i in range(e.layers)])
            self.layer_norm = None
        elif e.layer_type == "transformer":
            self.layers = nn.ModuleList([_TransformerLayer(d, e.ffn_embed_dim, e.attention_heads, pos[i], rel)
                                         for i in range(e.layers)])
            self.layer_norm = _Affine(d)
        else:
            raise NotImplementedError(e.layer_type)
        self.vocab_size = vocab_size
        self.fc_out = _Linear(d, vocab_size, xavier=1.0) if vocab_size is not None else None
        # limited self-attention context, "(left, right)" in frames (speech_transformer_encoder.py:179-190)
        ctx_ = e.transformer_context
        if isinstance(ctx_, str):
            ctx_ = eval_str_nested_list_or_tuple(ctx_, type=int)
        if ctx_ is not None:
            if len(ctx_) != 2 or any(c is not None and (not isinstance(c, int) or c < 0) for c in ctx_):
                raise ValueError("transformer_context must be a pair of None / non-negative ints, got %r" % (ctx_,))
            ctx_ = tuple(ctx_)
        self.transformer_context = ctx_
        self.num_updates = 0
        self.flat = None
        self.flat_prefix = ""
        self.engine = None
        self._anchor = None
        self.dropout_seed = 1

    # ---- native wiring ----------------------------------------------------------------------------
    def flat_groups(self, prefix=""):
        """Parameters that must be adjacent in the flat buffer (fused QKV views)."""
        groups = []
        for i in range(len(self.layers)):
            groups.append([prefix + "layers.%d.self_attn.%s_proj.weight" % (i, c) for c in "qkv"])
            groups.append([prefix + "layers.%d.self_attn.%s_proj.bias" % (i, c) for c in "qkv"])
        return groups

    def channels_last_params(self, prefix=""):
        return [] if self.pre_encoder is None else self.pre_encoder.channels_last_weights(prefix + "pre_encoder.")

    def finalize_(self, device, flat=None, prefix=""):
        """Cast to bf16 on `device`, re-home all parameters into the flat buffers and build the engine.
        Call once after construction / load_state_dict (fairseq does the equivalent cast in
        fairseq/trainer.py:105-107).  `flat`/`prefix`: a FlatParams built by the owning model over
        encoder + decoder (the parameters of this module are then named prefix + local name)."""
        self.to(device)
        if flat is None:
            flat = FlatParams(self, groups=self.flat_groups(), device=device, channels_last=self.channels_last_params())
        self.flat, self.flat_prefix = flat, prefix
        if self.pre_encoder is not None:
            self.pre_encoder.use_flat_(flat, prefix + "pre_encoder.")
        e = self.cfg.encoder
        ecfg = dict(embed_dim=e.embed_dim, ffn_dim=e.ffn_embed_dim, heads=e.attention_heads, layers=e.layers,
                    layer_type=e.layer_type, dw_kernel=e.depthwise_conv_kernel_size, dropout=self.cfg.dropout,
                    attention_dropout=self.cfg.attention_dropout, activation_dropout=self.cfg.activation_dropout,
                    layernorm_embedding=self.cfg.layernorm_embedding, final_layer_norm=self.layer_norm is not None,
                    vocab=self.vocab_size, rel_pos=e.relative_positional_embeddings)
        if e.relative_positional_embeddings and e.learned_pos:
            # layer -> flat name of its table (a table shared across layers is registered once)
            seen = {}
            ecfg["learned_pos_tables"] = {
                i: seen.setdefault(id(l.self_attn.positional_embedding.weight),
                                   prefix + "layers.%d.self_attn.positional_embedding.weight" % i)
                for i, l in enumerate(self.layers)}
        self.engine = EncoderEngine(self.flat, prefix, ecfg)
        if e.layer_type == "conformer":
            self.engine.bn_state = {i: (l.conv_module.batch_norm.running_mean, l.conv_module.batch_norm.running_var)
                                    for i, l in enumerate(self.layers)}
            for l in self.layers:
                l.conv_module.batch_norm.fp32_running_stats_()
        self._anchor = torch.zeros(1, device=device, requires_grad=True)
        return self

    def sync_torch_grads_(self):
        """Fold the gradients of the torch-executed conv front (bf16 .grad) into the flat fp32 buffer."""
        if self.pre_encoder is not None:
            self.flat.fold_torch_grads_(self.pre_encoder, self.flat_prefix + "pre_encoder.")

    def set_num_updates(self, num_updates):
        self.num_updates = num_updates

    def output_lengths(self, in_lengths):
        return in_lengths if self.pre_encoder is None else self.pre_encoder.output_lengths(in_lengths)

    def max_positions(self):
        return self.max_source_positions

    @property
    def has_attn_mask(self):
        c = self.transformer_context
        return self.cfg.encoder.chunk_size > 0 or (c is not None and (c[0] is not None or c[1] is not None))

    def attn_key_bounds(self, max_len, T):
        """The reference's get_attn_mask (speech_transformer_encoder.py:226-263) as per-row key ranges: numpy int32
        (lo, hi) of length T, or None.  Chunk streaming takes precedence over transformer_context, and its first-or-last
        partial chunk coin is drawn under numpy_seed(num_updates) exactly like the reference."""
        e = self.cfg.encoder
        if e.chunk_size > 0:
            with numpy_seed(self.num_updates):
                lo, hi = chunk_streaming_bounds(max_len, e.chunk_size, e.chunk_left_window, e.chunk_right_window,
                                                always_partial_in_last=not self.training)
        elif self.has_attn_mask:
            lo, hi = context_bounds(max_len, *self.transformer_context)
        else:
            return None
        if T > max_len:  # rows beyond the longest utterance (shape bucketing) are padding: any non-empty range does
            lo = np.concatenate([lo, np.zeros(T - max_len, np.int32)])
            hi = np.concatenate([hi, np.full(T - max_len, max_len, np.int32)])
        return lo, hi

    def forward(self, src_tokens, src_lengths, return_all_hiddens: bool = False, src_lengths_cpu=None):
        if self.engine is None:
            raise RuntimeError("call finalize_(device) before running the native encoder")
        x = src_tokens
        if x.dtype != torch.bfloat16:
            x = x.to(torch.bfloat16)  # fairseq/trainer.py:1279-1297 casts float samples under --bf16
        if self.pre_encoder is not None:
            x, out_lens = self.pre_encoder(x, src_lengths)
        else:
            out_lens = src_lengths
        B, T, _ = x.shape
        lens_cpu = src_lengths_cpu if src_lengths_cpu is not None else src_lengths.cpu()
        out_lens_cpu = self.output_lengths(lens_cpu)
        has_pads = bool((out_lens_cpu < T).any())
        lens_i32 = out_lens.to(torch.int32)
        eng = self.engine
        eng.training = self.training
        # per-update variation comes from the device seed tensor when a trainer installed one (graph-replay safe)
        eng.seed = self.dropout_seed if _ops._SEED_T is not None else self.dropout_seed * 7919 + self.num_updates
        eng.key_bounds = None
        if self.has_attn_mask:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError("streaming / limited-context attention masks change per update; run without CUDA graphs")
            lo, hi = self.attn_key_bounds(int(out_lens_cpu.max()), T)
            eng.key_bounds = (torch.from_numpy(lo).to(x.device, non_blocking=True),
                              torch.from_numpy(hi).to(x.device, non_blocking=True))
        if self.training:
            for l in self.layers:
                if hasattr(l, "conv_module"):
                    l.conv_module.batch_norm.num_batches_tracked += 1
        if torch.is_grad_enabled() and self.training:
            out = _EncoderFn.apply(x.contiguous(), self._anchor, eng, lens_i32, has_pads)
        else:
            out = eng.forward(x.contiguous(), lens_i32, has_pads, save=False)
        V = self.vocab_size
        pad_mask = torch.arange(T, device=x.device)[None, :] >= out_lens[:, None]
        enc_out = out[:, :, :V] if V is not None else out
        return {
            "encoder_out": [enc_out.transpose(0, 1)],  # T x B x C (a view of the batch-major buffer)
            "encoder_padding_mask": [pad_mask] if has_pads else [],
            "encoder_embedding": [],
            "encoder_states": [],
            "fc_results": [],
            "src_tokens": [],
            "src_lengths": [out_lens],
            "b200_out": out,  # batch-major [B, T', ld] buffer the native criterions consume directly
        }


def encoder_inputs(model, src_tokens, src_lengths, src_lengths_cpu=None, freq_masks=None, time_masks=None, time_warp=None):
    """A batch as the encoder takes it: (features [B, T, F], lengths, host lengths or None).  The SpecAugment descriptors
    (time warp, frequency and time masks) apply in training only.  Features [B, T, F] pass through, or through
    esp_specaug_features when descriptors are given.  Raw waveforms [B, N] (int16 range, lengths in samples) go through
    `model.frontend`, and host lengths in samples become frame counts."""
    if not model.training:
        freq_masks = time_masks = time_warp = None
    if src_tokens.dim() != 2:
        if freq_masks is not None or time_masks is not None or time_warp is not None:
            src_tokens = _ops.specaug_features(src_tokens, src_lengths.to(torch.int32), time_warp, freq_masks, time_masks)
        return src_tokens, src_lengths, src_lengths_cpu
    if getattr(model, "frontend", None) is None:
        raise RuntimeError("raw waveform input needs model.frontend (espresso_b200.data.frontend.OnTheFlyFbank)")
    if time_warp is None:
        feats, lens = model.frontend(src_tokens, src_lengths, freq_masks, time_masks)
    else:
        feats, lens = model.frontend(src_tokens, src_lengths, freq_masks, time_masks, time_warp=time_warp)
    return feats, lens, None if src_lengths_cpu is None else _ops.num_frames(src_lengths_cpu)


@register_model("speech_transformer_encoder_model", dataclass=SpeechTransformerConfig)
class SpeechTransformerEncoderModel(nn.Module):
    def __init__(self, cfg, encoder):
        super().__init__()
        self.cfg = cfg
        self.encoder = encoder
        self.num_updates = 0
        self.frontend = None  # optional espresso_b200.data.frontend.OnTheFlyFbank (not a submodule: no parameters)

    @classmethod
    def build_model(cls, cfg, task):
        """speech_transformer_encoder_model.py:50-117: needs task.feat_dim, task.feat_in_channels,
        task.target_dictionary."""
        if cfg.max_source_positions is None:
            cfg.max_source_positions = DEFAULT_MAX_SOURCE_POSITIONS
        e = cfg.encoder
        conv, size = ConvBNReLU.from_config(e.conv_channels, e.conv_kernel_sizes, e.conv_strides, task.feat_dim,
                                            task.feat_in_channels)
        vocab = len(task.target_dictionary) if task.target_dictionary is not None else None
        encoder = SpeechTransformerEncoderForPrediction(cfg, pre_encoder=conv, input_size=size, vocab_size=vocab)
        return cls(cfg, encoder)

    def sync_torch_grads_(self):
        self.encoder.sync_torch_grads_()

    def finalize_(self, device):
        self.to(device)
        flat = FlatParams(self, groups=self.encoder.flat_groups("encoder."), device=device,
                          channels_last=self.encoder.channels_last_params("encoder."))
        self.encoder.finalize_(device, flat=flat, prefix="encoder.")
        return self

    @property
    def flat(self):
        return self.encoder.flat

    def set_num_updates(self, num_updates):
        self.num_updates = num_updates
        self.encoder.set_num_updates(num_updates)

    def output_lengths(self, in_lengths):
        return self.encoder.output_lengths(in_lengths)

    def max_positions(self):
        return self.encoder.max_positions()

    def forward(self, src_tokens, src_lengths, freq_masks=None, time_masks=None, src_lengths_cpu=None, time_warp=None,
                **kwargs):
        """src_tokens: features [B, T, F] (reference layout) or, with the on-device front end, raw waveforms
        [B, N] in int16 range with src_lengths = sample counts (+ host-drawn SpecAugment descriptors)."""
        x, lens, lens_cpu = encoder_inputs(self, src_tokens, src_lengths, src_lengths_cpu, freq_masks, time_masks,
                                           time_warp)
        return self.encoder(x, lens, src_lengths_cpu=lens_cpu)

    def get_normalized_probs(self, net_output, log_probs, sample=None):
        """fp32 (log-)softmax over the vocabulary (speech_transformer_encoder_model.py:141-150).  Used by the
        validation decoders; the native CTC criterion never materialises this tensor."""
        logits = net_output["encoder_out"][0].float()
        return F.log_softmax(logits, dim=-1) if log_probs else F.softmax(logits, dim=-1)
