"""Oracle: speech Transformer/Conformer encoder (+ CTC criterion) as plain functional PyTorch.

TEST INFRASTRUCTURE ONLY (also the CPU `--impl reference` arm of bench.py).  A restatement -- written
against the reference's behaviour, operating directly on a state_dict with the reference's parameter
names -- of:
  espresso/modules/speech_convolutions.py:78-102                         conv_front
  espresso/models/transformer/speech_transformer_encoder.py:298-409     encoder_forward
  espresso/modules/conformer_with_relative_positional_embedding_encoder_layer.py:81-145   conformer_layer
  fairseq/modules/conformer_layer.py:79-101,134-146                      conv_module / ffn_module
  fairseq/modules/multihead_attention.py:639-917 (rel-pos branch)        relpos_mha
  espresso/modules/sinusoidal_relative_positional_embedding.py:46-124    rel_pos_table
  fairseq/modules/transformer_layer.py:163-226                           transformer_layer
  espresso/models/transformer/speech_transformer_encoder_model.py:141-150,177-210   fc_out / log-softmax
  espresso/criterions/ctc_loss.py:59-103                                 ctc_criterion
Pinned against the real reference by oracle/pin_against_reference.py (section "conformer").
"""
import math

import torch
import torch.nn.functional as F

DEFAULT_STRIDES = ((1, 1), (2, 2), (1, 1), (2, 2))


def out_lengths(lens, strides=DEFAULT_STRIDES):
    for s in strides:
        lens = (lens + s[0] - 1) // s[0]
    return lens


def rel_pos_table(T, d, dtype=torch.float32):
    half = d // 2
    freq = torch.exp(torch.arange(half, dtype=torch.float32) * -(math.log(10000.0) / (half - 1)))
    pos = torch.arange(-(T - 1), T, dtype=torch.float32)[:, None] * freq[None, :]
    emb = torch.cat([torch.sin(pos), torch.cos(pos)], dim=1)
    if d % 2 == 1:
        emb = torch.cat([emb, torch.zeros(emb.shape[0], 1)], dim=1)
    return (emb * d ** -0.5).to(dtype)


def _drop(x, p, training, site, masks=None):
    """Dropout at the named site (parameter prefix + role: ffn.act, ffn.out, attn.probs, mha.out, conv.out, front.out,
    embed.out).  masks: optional provider masks(site, x) -> fp32 multiplier of x's shape (keep / (1 - p), else 0); it
    replaces F.dropout's own draw, so a model run can be replayed with the masks of another implementation."""
    if not (training and p > 0):
        return x
    if masks is None:
        return F.dropout(x, p, training)
    return x * masks(site, x).to(x.dtype)


def conv_front(sd, pre, x, lens, strides, training):
    """x [B, T, F] -> ([B, T', C*F'], out_lens, padding_mask [B, T'])."""
    B, T, Fd = x.shape
    h = x.view(B, T, 1, Fd).transpose(1, 2)
    for i, s in enumerate(strides):
        h = F.conv2d(h, sd[pre + "convolutions.%d.weight" % i], sd[pre + "convolutions.%d.bias" % i], stride=s, padding=1)
        bn = pre + "batchnorms.%d." % i
        h = F.batch_norm(h, sd[bn + "running_mean"], sd[bn + "running_var"], sd[bn + "weight"], sd[bn + "bias"],
                         training, 0.1, 1e-5)
        h = F.relu(h)
    h = h.transpose(1, 2).contiguous()
    h = h.view(h.size(0), h.size(1), -1)
    ol = out_lengths(lens, strides)
    pad = torch.arange(h.size(1), device=x.device)[None, :] >= ol[:, None]
    if pad.any():
        h = h.masked_fill(pad[:, :, None], 0.0)
    return h, ol, pad


def relpos_mha(sd, p, x, pad_mask, H, attn_drop, training, attn_mask=None, masks=None):
    """x [B, T, d] (batch-major here; the reference is time-major, the math is identical)."""
    B, T, d = x.shape
    hd = d // H
    s = hd ** -0.5
    q = F.linear(x, sd[p + "q_proj.weight"], sd[p + "q_proj.bias"])
    k = F.linear(x, sd[p + "k_proj.weight"], sd[p + "k_proj.bias"])
    v = F.linear(x, sd[p + "v_proj.weight"], sd[p + "v_proj.bias"])
    kh = k.view(B, T, H, hd).transpose(1, 2)
    vh = v.view(B, T, H, hd).transpose(1, 2)
    if p + "positional_embedding.weight" in sd:
        # learned relative positions (espresso/modules/learned_relative_positional_embedding.py:47-88 +
        # multihead_attention.py:799-823 with `learnable`): no pos_bias_u/v, no pos_proj; the table has
        # 2*max_size-1 rows of width d or head_dim (shared across heads), rows max_size-T .. max_size+T-2 are used
        tab = sd[p + "positional_embedding.weight"]
        n_emb, E = tab.shape
        pos = torch.arange(n_emb // 2 - T + 1, n_emb // 2 + T, device=x.device).clamp(0, n_emb - 1)
        pe = tab[pos]                                                           # [2T-1, E]
        qu = qv = (q * s).view(B, T, H, hd).transpose(1, 2)
        ph = (pe[:, None, :].expand(-1, H, -1) if E == hd else pe.view(2 * T - 1, H, hd)).permute(1, 2, 0)
    else:
        qv = ((q + sd[p + "pos_bias_v"]) * s).view(B, T, H, hd).transpose(1, 2)   # [B,H,T,hd]
        qu = ((q + sd[p + "pos_bias_u"]) * s).view(B, T, H, hd).transpose(1, 2)
        pe = F.linear(rel_pos_table(T, d, x.dtype).to(x.device), sd[p + "pos_proj.weight"])  # [2T-1, d]
        ph = pe.view(2 * T - 1, H, hd).permute(1, 2, 0)                             # [H, hd, 2T-1]
    ac = qu @ kh.transpose(-1, -2)                                             # [B,H,T,T]
    bd_full = qv @ ph[None]                                                     # [B,H,T,2T-1]
    i = torch.arange(T, device=x.device)[:, None]
    j = torch.arange(T, device=x.device)[None, :]
    bd = bd_full.gather(-1, ((T - 1) - i + j).expand(B, H, T, T))               # skew: r = j - i
    w = ac + bd
    if attn_mask is not None:   # [T, T] additive mask (multihead_attention.py:835-839)
        w = w + attn_mask.to(w.dtype)
    if pad_mask is not None:
        w = w.masked_fill(pad_mask[:, None, None, :], float("-inf"))
    w = torch.softmax(w.float(), dim=-1).to(w.dtype)
    w = _drop(w, attn_drop, training, p + "attn.probs", masks)
    ctx = (w @ vh).transpose(1, 2).reshape(B, T, d)
    return F.linear(ctx, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"])


def ffn_module(sd, p, x, act_drop, drop, training, masks=None):
    h = F.layer_norm(x, (x.size(-1),), sd[p + "layer_norm.weight"], sd[p + "layer_norm.bias"])
    h = F.silu(F.linear(h, sd[p + "w_1.weight"], sd[p + "w_1.bias"]))
    h = _drop(h, act_drop, training, p + "ffn.act", masks)
    h = F.linear(h, sd[p + "w_2.weight"], sd[p + "w_2.bias"])
    return _drop(h, drop, training, p + "ffn.out", masks)


def conv_module(sd, p, x, drop, training, masks=None):
    """x [B, T, d]; BatchNorm uses batch statistics over ALL B*T positions, padded ones included."""
    d = x.size(-1)
    h = F.layer_norm(x, (d,), sd[p + "layer_norm.weight"], sd[p + "layer_norm.bias"]).transpose(1, 2)
    h = F.glu(F.conv1d(h, sd[p + "pointwise_conv1.weight"]), dim=1)
    wd = sd[p + "depthwise_conv.weight"]
    h = F.conv1d(h, wd, padding=(wd.size(-1) - 1) // 2, groups=d)
    h = F.batch_norm(h, sd[p + "batch_norm.running_mean"], sd[p + "batch_norm.running_var"], sd[p + "batch_norm.weight"],
                     sd[p + "batch_norm.bias"], training, 0.1, 1e-5)
    h = F.conv1d(F.silu(h), sd[p + "pointwise_conv2.weight"])
    if masks is not None:  # providers see batch-major [B, T, d] activations
        return _drop(h.transpose(1, 2), drop, training, p + "conv.out", masks)
    return _drop(h, drop, training, p + "conv.out").transpose(1, 2)


def conformer_layer(sd, p, x, pad_mask, cfg, training, attn_mask=None):
    dr, adr, acdr = cfg["dropout"], cfg["attention_dropout"], cfg["activation_dropout"]
    mk = cfg.get("dropout_masks")
    x = x + 0.5 * ffn_module(sd, p + "ffn1.", x, acdr, dr, training, mk)
    h = F.layer_norm(x, (x.size(-1),), sd[p + "self_attn_layer_norm.weight"], sd[p + "self_attn_layer_norm.bias"])
    x = x + _drop(relpos_mha(sd, p + "self_attn.", h, pad_mask, cfg["heads"], adr, training, attn_mask, mk), dr, training,
                  p + "mha.out", mk)
    x = x + conv_module(sd, p + "conv_module.", x, dr, training, mk)
    x = x + 0.5 * ffn_module(sd, p + "ffn2.", x, acdr, dr, training, mk)
    return F.layer_norm(x, (x.size(-1),), sd[p + "final_layer_norm.weight"], sd[p + "final_layer_norm.bias"])


def transformer_layer(sd, p, x, pad_mask, cfg, training, attn_mask=None):
    dr, adr, acdr = cfg["dropout"], cfg["attention_dropout"], cfg["activation_dropout"]
    mk = cfg.get("dropout_masks")
    h = F.layer_norm(x, (x.size(-1),), sd[p + "self_attn_layer_norm.weight"], sd[p + "self_attn_layer_norm.bias"])
    x = x + _drop(relpos_mha(sd, p + "self_attn.", h, pad_mask, cfg["heads"], adr, training, attn_mask, mk), dr, training,
                  p + "mha.out", mk)
    h = F.layer_norm(x, (x.size(-1),), sd[p + "final_layer_norm.weight"], sd[p + "final_layer_norm.bias"])
    h = _drop(F.relu(F.linear(h, sd[p + "fc1.weight"], sd[p + "fc1.bias"])), acdr, training, p + "ffn.act", mk)
    return x + _drop(F.linear(h, sd[p + "fc2.weight"], sd[p + "fc2.bias"]), dr, training, p + "ffn.out", mk)


def encoder_forward(sd, cfg, feats, lens, training=False, pre="encoder.", skip_conv_front=False, attn_mask=None):
    """feats [B, T, 80] (or the conv-front output if skip_conv_front), lens [B] ->
    (out [B, T', V or d], out_lens, padding_mask).  cfg["dropout_masks"] (optional): mask provider of _drop.  attn_mask: optional [T', T'] bool, True = HIDDEN key
    (speech_transformer_encoder.py:368-379; the layers turn it into an additive -1e8 / -1e4 mask)."""
    if skip_conv_front:
        x, ol = feats, lens
        pad = torch.arange(x.size(1), device=x.device)[None, :] >= ol[:, None]
    else:
        x, ol, pad = conv_front(sd, pre + "pre_encoder.", feats, lens, cfg.get("strides", DEFAULT_STRIDES), training)
    has_pads = bool(pad.any())
    mk = cfg.get("dropout_masks")
    x = _drop(x, cfg["dropout"], training, pre + "front.out", mk)
    x = F.linear(x, sd[pre + "fc0.weight"], sd[pre + "fc0.bias"])
    if cfg.get("layernorm_embedding", False):
        x = F.layer_norm(x, (x.size(-1),), sd[pre + "layernorm_embedding.weight"], sd[pre + "layernorm_embedding.bias"])
    x = _drop(x, cfg["dropout"], training, pre + "embed.out", mk)
    if has_pads:
        x = x * (~pad)[:, :, None].to(x.dtype)
    layer_fn = conformer_layer if cfg["layer_type"] == "conformer" else transformer_layer
    # transformer_layer.py:189-192 / conformer_with_relative_positional_embedding_encoder_layer.py:107-110
    add_mask = None if attn_mask is None else attn_mask.to(x.dtype).masked_fill(
        attn_mask, -1e8 if x.dtype == torch.float32 else -1e4)
    for i in range(cfg["layers"]):
        x = layer_fn(sd, pre + "layers.%d." % i, x, pad if has_pads else None, cfg, training, add_mask)
    if cfg.get("final_layer_norm", False):
        x = F.layer_norm(x, (x.size(-1),), sd[pre + "layer_norm.weight"], sd[pre + "layer_norm.bias"])
    if cfg.get("vocab"):
        x = F.linear(x, sd[pre + "fc_out.weight"], sd[pre + "fc_out.bias"])
    return x, ol, pad


def ctc_criterion(logits, out_lens, target, pad_idx, eos_idx, blank_idx, zero_infinity=True):
    """logits [B, T', V]; target [B, U] with pad/eos -> summed CTC loss (espresso/criterions/ctc_loss.py:59-103)."""
    lprobs = F.log_softmax(logits.float(), dim=-1).transpose(0, 1)
    keep = (target != pad_idx) & (target != eos_idx)
    flat = target[keep]
    tl = keep.sum(-1)
    return F.ctc_loss(lprobs, flat, out_lens.long(), tl, blank=blank_idx, reduction="sum", zero_infinity=zero_infinity)


def random_state_dict(cfg, seed=1, feat_dim=80, conv_channels=(64, 64, 128, 128), dtype=torch.float32):
    """A random parameter set with the reference's names/shapes (for benchmarks and self-consistency tests)."""
    g = torch.Generator().manual_seed(seed)
    d, ffn, L, V = cfg["embed_dim"], cfg["ffn_dim"], cfg["layers"], cfg.get("vocab")

    def rnd(*shape, scale=None):
        fan_in = shape[-1] if len(shape) > 1 else shape[0]
        sc = scale if scale is not None else (1.0 / math.sqrt(fan_in))
        return ((torch.rand(*shape, generator=g) * 2 - 1) * sc * math.sqrt(3.0)).to(dtype)

    sd = {}
    pre = "encoder."
    cin, fd = 1, feat_dim
    for i, (c, s) in enumerate(zip(conv_channels, cfg.get("strides", DEFAULT_STRIDES))):
        sd[pre + "pre_encoder.convolutions.%d.weight" % i] = rnd(c, cin, 3, 3, scale=1.0 / math.sqrt(cin * 9))
        sd[pre + "pre_encoder.convolutions.%d.bias" % i] = rnd(c, scale=0.05)
        bn = pre + "pre_encoder.batchnorms.%d." % i
        sd[bn + "weight"] = 1.0 + rnd(c, scale=0.1)
        sd[bn + "bias"] = rnd(c, scale=0.1)
        sd[bn + "running_mean"] = torch.zeros(c, dtype=dtype)
        sd[bn + "running_var"] = torch.ones(c, dtype=dtype)
        cin = c
        fd = (fd + s[1] - 1) // s[1]
    sd[pre + "fc0.weight"] = rnd(d, cin * fd)
    sd[pre + "fc0.bias"] = rnd(d, scale=0.02)
    if cfg.get("layernorm_embedding", False):
        sd[pre + "layernorm_embedding.weight"] = 1.0 + rnd(d, scale=0.1)
        sd[pre + "layernorm_embedding.bias"] = rnd(d, scale=0.1)

    def ln(name):
        sd[name + ".weight"] = 1.0 + rnd(d, scale=0.1)
        sd[name + ".bias"] = rnd(d, scale=0.1)

    for i in range(L):
        p = pre + "layers.%d." % i
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            sd[p + "self_attn.%s.weight" % nm] = rnd(d, d)
            sd[p + "self_attn.%s.bias" % nm] = rnd(d, scale=0.02)
        sd[p + "self_attn.pos_bias_u"] = rnd(d, scale=0.1)
        sd[p + "self_attn.pos_bias_v"] = rnd(d, scale=0.1)
        sd[p + "self_attn.pos_proj.weight"] = rnd(d, d)
        ln(p + "self_attn_layer_norm")
        ln(p + "final_layer_norm")
        if cfg["layer_type"] == "conformer":
            for f in ("ffn1", "ffn2"):
                ln(p + f + ".layer_norm")
                sd[p + f + ".w_1.weight"] = rnd(ffn, d)
                sd[p + f + ".w_1.bias"] = rnd(ffn, scale=0.02)
                sd[p + f + ".w_2.weight"] = rnd(d, ffn)
                sd[p + f + ".w_2.bias"] = rnd(d, scale=0.02)
            c = p + "conv_module."
            ln(c + "layer_norm")
            sd[c + "pointwise_conv1.weight"] = rnd(2 * d, d, 1, scale=1.0 / math.sqrt(d))
            k = cfg.get("dw_kernel", 31)
            sd[c + "depthwise_conv.weight"] = rnd(d, 1, k, scale=1.0 / math.sqrt(k))
            sd[c + "batch_norm.weight"] = 1.0 + rnd(d, scale=0.1)
            sd[c + "batch_norm.bias"] = rnd(d, scale=0.1)
            sd[c + "batch_norm.running_mean"] = torch.zeros(d, dtype=dtype)
            sd[c + "batch_norm.running_var"] = torch.ones(d, dtype=dtype)
            sd[c + "pointwise_conv2.weight"] = rnd(d, d, 1, scale=1.0 / math.sqrt(d))
        else:
            sd[p + "fc1.weight"] = rnd(ffn, d)
            sd[p + "fc1.bias"] = rnd(ffn, scale=0.02)
            sd[p + "fc2.weight"] = rnd(d, ffn)
            sd[p + "fc2.bias"] = rnd(d, scale=0.02)
    if cfg.get("final_layer_norm", False):
        ln(pre + "layer_norm")
    if V:
        sd[pre + "fc_out.weight"] = rnd(V, d)
        sd[pre + "fc_out.bias"] = rnd(V, scale=0.02)
    return sd
