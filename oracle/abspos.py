"""Oracle: encoders with ABSOLUTE positions (relative positional embeddings off) and relaxed encoder-decoder attention,
as plain functional PyTorch on a state_dict with the reference's parameter names.  TEST INFRASTRUCTURE ONLY.  Restates:
  fairseq/modules/sinusoidal_positional_embedding.py + speech_transformer_encoder.py:93-101,341-345   abs_positions
  fairseq/modules/multihead_attention.py:639-917 (plain branch)                                      plain_mha
  fairseq/modules/multihead_attention.py:869-872 (relaxed attention, training only)                  decoder_mha
and the per-op statements of the kernels' new entry points (attention without positions, the backward without the
skewed copy, relaxed probabilities), on top of oracle/ops_ref.py.  The layer / conv-front / loss pieces are the ones of
oracle/conformer.py and oracle/decoder.py.  Pinned against the real reference by oracle/pin_abspos.py.

The fixtures store no parameters: both the reference (at pinning time) and the tests fill the model's state dict with
`seeded_state_dict`, a deterministic function of each tensor's name and shape.  Nor do they store the reference's
gradients: they store a sketch of each (its norm and projections on seeded unit vectors, `grad_sketch`), against which
the oracle's gradients are checked; the native paths are then compared with the oracle's full gradients."""
import math
import zlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import conformer as OC
from oracle import decoder as OD
from oracle import ops_ref

BF = torch.bfloat16


# ---------------------------------------------------------------------------------------------------
# parameters and gradient sketches
# ---------------------------------------------------------------------------------------------------
def _gen(name, seed):
    return torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(name.encode())) & 0x7FFFFFFF)


def seeded_state_dict(shapes, seed=1):
    """{name: shape} -> {name: tensor}: uniform weights at 1/sqrt(fan_in), LayerNorm / BatchNorm scales 1 +- 0.1, biases
    and position biases +- 0.1, BatchNorm running statistics (0, 1), buffers as the reference initialises them."""
    sd = {}
    for name, shape in shapes.items():
        shape = tuple(shape)
        if name.endswith("num_batches_tracked"):
            sd[name] = torch.zeros(shape, dtype=torch.long)
            continue
        if name.endswith("running_mean") or name.endswith("_float_tensor"):
            sd[name] = torch.zeros(shape)
            continue
        if name.endswith("running_var"):
            sd[name] = torch.ones(shape)
            continue
        if name.endswith("version"):
            sd[name] = torch.full(shape, 3.0)
            continue
        u = torch.rand(shape, generator=_gen(name, seed)) * 2 - 1
        if len(shape) == 1:
            norm_scale = name.endswith(".weight") and ("norm" in name or "batchnorms" in name)
            sd[name] = 1.0 + 0.1 * u if norm_scale else 0.1 * u
        else:
            fan_in = int(np.prod(shape[1:]))
            sd[name] = u * math.sqrt(3.0 / fan_in)
    return sd


SKETCH_K = 8


def grad_sketch(name, g):
    """[norm, K projections on seeded unit vectors] of one gradient (float64)."""
    x = g.detach().double().reshape(-1)
    r = torch.randn(SKETCH_K, x.numel(), generator=_gen("sketch." + name, 7), dtype=torch.float64)
    r = r / r.norm(dim=1, keepdim=True)
    return np.concatenate([[x.norm().item()], (r @ x).numpy()])


def sketch_error(name, g, sketch):
    """Largest deviation of g's sketch from a recorded one, relative to the recorded norm (floor 1e-3)."""
    s = grad_sketch(name, g)
    return float(np.abs(s - sketch).max() / max(sketch[0], 1e-3))


def skip_grad(name):
    """Analytically zero gradients (bias in front of a batch-statistics BatchNorm; key bias under softmax): the reference
    back-propagates rounding noise into them."""
    return ("pre_encoder.convolutions" in name and name.endswith(".bias")) or name.endswith("k_proj.bias")


# ---------------------------------------------------------------------------------------------------
# model pieces
# ---------------------------------------------------------------------------------------------------
def abs_positions(pad_mask, d, dtype=torch.float32):
    """embed_positions((~pad).int()) with fairseq's sinusoidal table and padding_idx 0: valid frame t reads row t + 1
    (make_positions: cumsum of the non-padding mask), padded frames the zero row 0.  pad_mask [B, T] bool -> [B, T, d]."""
    B, T = pad_mask.shape
    nonpad = (~pad_mask).long()
    positions = torch.cumsum(nonpad, dim=1) * nonpad
    return OD.sinusoidal_table(T + 1, d, 0).to(dtype)[positions]


def plain_mha(sd, p, x, pad_mask, H):
    """Plain scaled dot-product self-attention: q = q_proj(x) * scaling, softmax(q k^T + key padding) v (dropout 0)."""
    B, T, d = x.shape
    hd = d // H
    q = (F.linear(x, sd[p + "q_proj.weight"], sd[p + "q_proj.bias"]) * hd ** -0.5).view(B, T, H, hd).transpose(1, 2)
    kh = F.linear(x, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"]).view(B, T, H, hd).transpose(1, 2)
    vh = F.linear(x, sd[p + "v_proj.weight"], sd[p + "v_proj.bias"]).view(B, T, H, hd).transpose(1, 2)
    w = q @ kh.transpose(-1, -2)
    if pad_mask is not None:
        w = w.masked_fill(pad_mask[:, None, None, :], float("-inf"))
    w = torch.softmax(w.float(), dim=-1).to(w.dtype)
    ctx = (w @ vh).transpose(1, 2).reshape(B, T, d)
    return F.linear(ctx, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"])


def _layer_norm(sd, p, x):
    return F.layer_norm(x, (x.size(-1),), sd[p + ".weight"], sd[p + ".bias"])


def conformer_layer(sd, p, x, pad_mask, cfg, training):
    """conformer_with_relative_positional_embedding_encoder_layer.py:81-145 with the plain attention (dropout 0)."""
    x = x + 0.5 * OC.ffn_module(sd, p + "ffn1.", x, 0.0, 0.0, training)
    x = x + plain_mha(sd, p + "self_attn.", _layer_norm(sd, p + "self_attn_layer_norm", x), pad_mask, cfg["heads"])
    x = x + OC.conv_module(sd, p + "conv_module.", x, 0.0, training)
    x = x + 0.5 * OC.ffn_module(sd, p + "ffn2.", x, 0.0, 0.0, training)
    return _layer_norm(sd, p + "final_layer_norm", x)


def transformer_layer(sd, p, x, pad_mask, cfg, training):
    """Pre-LN transformer_layer.py:163-226 with the plain attention (dropout 0)."""
    x = x + plain_mha(sd, p + "self_attn.", _layer_norm(sd, p + "self_attn_layer_norm", x), pad_mask, cfg["heads"])
    h = F.relu(F.linear(_layer_norm(sd, p + "final_layer_norm", x), sd[p + "fc1.weight"], sd[p + "fc1.bias"]))
    return x + F.linear(h, sd[p + "fc2.weight"], sd[p + "fc2.bias"])


def encoder_forward(sd, cfg, feats, lens, training=False, pre="encoder."):
    """speech_transformer_encoder.py:298-409 with absolute positions (dropout 0): conv front, fc0, + positions,
    layernorm_embedding, padding mask, layers, final LayerNorm, fc_out.  -> (out [B, T', V or d], out_lens, pad)."""
    x, ol, pad = OC.conv_front(sd, pre + "pre_encoder.", feats, lens, OC.DEFAULT_STRIDES, training)
    x = F.linear(x, sd[pre + "fc0.weight"], sd[pre + "fc0.bias"])
    x = x + abs_positions(pad, x.size(-1), x.dtype)
    if cfg.get("layernorm_embedding", False):
        x = _layer_norm(sd, pre + "layernorm_embedding", x)
    has_pads = bool(pad.any())
    if has_pads:
        x = x * (~pad)[:, :, None].to(x.dtype)
    layer = conformer_layer if cfg["layer_type"] == "conformer" else transformer_layer
    for i in range(cfg["layers"]):
        x = layer(sd, pre + "layers.%d." % i, x, pad if has_pads else None, cfg, training)
    if cfg.get("final_layer_norm", False):
        x = _layer_norm(sd, pre + "layer_norm", x)
    if cfg.get("vocab"):
        x = F.linear(x, sd[pre + "fc_out.weight"], sd[pre + "fc_out.bias"])
    return x, ol, pad


def decoder_mha(sd, p, q_in, kv_in, H, key_pad, causal, relax=0.0):
    """oracle.decoder.mha (dropout 0) plus relaxed attention: (1 - relax) p + relax / Tk, Tk the PADDED key count."""
    B, Tq, d = q_in.shape
    Tk = kv_in.shape[1]
    hd = d // H
    q = (F.linear(q_in, sd[p + "q_proj.weight"], sd[p + "q_proj.bias"]) * hd ** -0.5).view(B, Tq, H, hd).transpose(1, 2)
    k = F.linear(kv_in, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"]).view(B, Tk, H, hd).transpose(1, 2)
    v = F.linear(kv_in, sd[p + "v_proj.weight"], sd[p + "v_proj.bias"]).view(B, Tk, H, hd).transpose(1, 2)
    w = q @ k.transpose(-1, -2)
    if causal:
        w = w + torch.triu(torch.full((Tq, Tk), float("-inf"), device=w.device), 1)
    if key_pad is not None:
        w = w.masked_fill(key_pad[:, None, None, :], float("-inf"))
    w = torch.softmax(w.float(), dim=-1).to(w.dtype)
    if relax > 0.0:
        w = (1.0 - relax) * w + relax / Tk
    ctx = (w @ v).transpose(1, 2).reshape(B, Tq, d)
    return F.linear(ctx, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"])


def decoder_forward(sd, cfg, prev_output_tokens, enc_out, enc_pad, training=False, pre="decoder."):
    """oracle.decoder.decoder_forward (dropout 0) with cfg["relaxed_attention_weight"] applied to the encoder attention in
    training (multihead_attention.py:869-872)."""
    pad = cfg["pad"]
    d, H = cfg["dec_embed_dim"], cfg["dec_heads"]
    relax = float(cfg.get("relaxed_attention_weight", 0.0)) if training else 0.0
    B, U = prev_output_tokens.shape
    x = math.sqrt(d) * F.embedding(prev_output_tokens, sd[pre + "embed_tokens.weight"], padding_idx=pad)
    nonpad = prev_output_tokens.ne(pad)
    positions = torch.cumsum(nonpad.long(), dim=1) * nonpad.long() + pad
    x = x + OD.sinusoidal_table(U + pad + 2, d, pad).to(x)[positions]
    tok_pad = prev_output_tokens.eq(pad)
    self_pad = tok_pad if bool(tok_pad.any()) else None
    for i in range(cfg["dec_layers"]):
        p = pre + "layers.%d." % i
        h = _layer_norm(sd, p + "self_attn_layer_norm", x)
        x = x + decoder_mha(sd, p + "self_attn.", h, h, H, self_pad, True)
        h = _layer_norm(sd, p + "encoder_attn_layer_norm", x)
        x = x + decoder_mha(sd, p + "encoder_attn.", h, enc_out, H, enc_pad, False, relax)
        h = F.relu(F.linear(_layer_norm(sd, p + "final_layer_norm", x), sd[p + "fc1.weight"], sd[p + "fc1.bias"]))
        x = x + F.linear(h, sd[p + "fc2.weight"], sd[p + "fc2.bias"])
    x = _layer_norm(sd, pre + "layer_norm", x)
    return F.linear(x, sd[pre + "output_projection.weight"])


def smoothed_ce(logits, target, pad, eps, smoothing, V):
    """label_smoothed_nll_loss (uniform or temporal, sum-reduced) through ops_ref.smoothing_weights -> (loss, nll)."""
    mode = ops_ref.SMOOTH_TEMPORAL if smoothing == "temporal" else ops_ref.SMOOTH_UNIFORM
    a, w = ops_ref.smoothing_weights(V, target.reshape(-1), pad, eps, mode, U=target.shape[1])
    lp = F.log_softmax(logits.float(), dim=-1).reshape(-1, V)
    keep = target.reshape(-1).ne(pad)
    nll = -lp.gather(1, target.reshape(-1, 1)).squeeze(1)[keep].sum()
    return a * nll + (w * -lp).sum(-1)[keep].sum(), nll


# ---------------------------------------------------------------------------------------------------
# per-op statements of the new entry points (same signatures as espresso_b200.ops)
# ---------------------------------------------------------------------------------------------------
def attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens, drop_p=0.0, seed=0, save_probs=True, pos_hstride=None, key_bounds=None):
    """ops_ref.attn_fused_fwd; pos None: the plain branch, s = qu k^T (qu = q * scaling), stated as the relative-position
    call with an all-zero table (S + bf16(0) is exact)."""
    if pos is None:
        hd = qu.shape[1] // H
        pos, qv, pos_hstride = torch.zeros(2 * T - 1, hd, dtype=BF), qu, 0
    return ops_ref.attn_fused_fwd(qu, qv, k, v, pos, B, T, H, lens, drop_p, seed, save_probs, pos_hstride, key_bounds)


def attn_fused_bwd(dctx, ctx, qu, v, p, pd, B, T, H, ldp, dk_out, dv_out, drop_p=0.0, seed=0):
    """ops_ref.attn_fused_bwd; ldp None: no skewed copy (returns dBD None)."""
    if ldp is not None:
        return ops_ref.attn_fused_bwd(dctx, ctx, qu, v, p, pd, B, T, H, ldp, dk_out, dv_out, drop_p, seed)
    ds, _ = ops_ref.attn_fused_bwd(dctx, ctx, qu, v, p, pd, B, T, H, (2 * T - 1 + 7) // 8 * 8, dk_out, dv_out, drop_p, seed)
    return ds, None


def attn_softmax_relaxed_fwd(scores, T, lens, relax_w, drop_p=0.0, seed=0):
    """Relaxed attention (multihead_attention.py:869-872): p = attn_softmax_fwd's P; p_drop = dropout(bf16(bf16((1 - w) p)
    + w / T)) over all T keys (the padded ones included), zeros in [T, ld).  1 - w and w / T are the reference's double
    scalars applied in fp32; dropout at index row * ld + j."""
    H, B, Tq, ld = scores.shape
    p, _ = ops_ref.attn_softmax_fwd(scores, T, lens)
    keep_w = torch.tensor(np.float32(1.0 - relax_w))
    add_w = torch.tensor(np.float32(relax_w / T))
    r = torch.zeros(H, B, Tq, ld)
    r[..., :T] = ((keep_w * p.float()[..., :T]).to(BF).float() + add_w).to(BF).float()
    if drop_p > 0:
        r = ops_ref._drop(r, drop_p, seed, ops_ref._flat_index(H, B, Tq, ld))
    return p, r.to(BF)


def cpu_ops():
    """{name: function}: every op of oracle/ops_ref.py with the three above in place of / beside its own, for
    monkeypatching espresso_b200.ops on the host."""
    table = {n: getattr(ops_ref, n) for n in dir(ops_ref) if not n.startswith("_") and callable(getattr(ops_ref, n))}
    table.update(attn_fused_fwd=attn_fused_fwd, attn_fused_bwd=attn_fused_bwd, attn_softmax_relaxed_fwd=attn_softmax_relaxed_fwd)
    return table
