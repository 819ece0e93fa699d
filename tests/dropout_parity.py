"""Shared by the CPU and GPU encoder-at-dropout tests: one training forward/backward of the native encoder model at
dropout = attention_dropout = activation_dropout = p, and the same step of the fp32 oracle model (oracle/conformer.py)
by autograd with the engine's own dropout masks injected at every site.

The oracle is bit-exact to the reference at dropout 0 and dropout only multiplies by a mask, so the oracle with the
engine's masks is the reference with those masks: any mismatch beyond bf16 rounding is a wrong seed, index or scale
somewhere in the engine's forward masks or in the masks its backward regenerates."""
import numpy as np
import torch

from oracle import conformer as OC
from oracle import dropout_rng as RNG

# oracle site role -> engine seed (layer, op) of espresso_b200/modules/encoder_engine.py; "L" = the layer index
CONFORMER_SEEDS = {"ffn1.ffn.act": ("L", 0), "ffn1.ffn.out": ("L", 1), "ffn2.ffn.act": ("L", 2), "ffn2.ffn.out": ("L", 3),
                   "self_attn.attn.probs": ("L", 10), "mha.out": ("L", 11), "conv_module.conv.out": ("L", 20)}
TRANSFORMER_SEEDS = {"ffn.act": ("L", 0), "ffn.out": ("L", 1), "self_attn.attn.probs": ("L", 10), "mha.out": ("L", 11)}
ENCODER_SEEDS = {"front.out": (999, 0), "embed.out": (999, 1)}


class _Dict:
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def pad(self):
        return 1

    def eos(self):
        return 2

    def index(self, sym):
        return 0


class _Task:
    feat_dim, feat_in_channels = 80, 1

    def __init__(self, V):
        self.target_dictionary = _Dict(V)


def case(golden_dir, layer_type, heads):
    """(sd, batch, dims) of one test case: the recorded toy fixture (d 64, 4 heads of width 16: the unfused attention
    path), or with heads=2 fresh oracle weights at d 128 (heads of width 64: the fused attention kernels) on the same
    padded batch."""
    import os

    g = np.load(os.path.join(golden_dir, "encoder_%s.npz" % layer_type))
    batch = {k: g[k] for k in ("feats", "lens", "target")}
    if heads == 4:
        return {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}, batch, dict(d=64, H=4)
    cfg = dict(embed_dim=128, ffn_dim=128, layers=2, layer_type=layer_type, dw_kernel=31, vocab=50, layernorm_embedding=True,
               final_layer_norm=layer_type != "conformer")
    return OC.random_state_dict(cfg, seed=7), batch, dict(d=128, H=heads)


def build(layer_type, sd, p, dev, d=64, H=4):
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel

    cfg = SpeechTransformerConfig.from_dict(dict(
        dropout=p, attention_dropout=p, activation_dropout=p, layernorm_embedding=True, max_source_positions=3600,
        encoder=dict(embed_dim=d, ffn_embed_dim=128, layers=2, attention_heads=H, normalize_before=True, learned_pos=False,
                     relative_positional_embeddings=True, layer_type=layer_type, depthwise_conv_kernel_size=31)))
    m = SpeechTransformerEncoderModel.build_model(cfg, _Task(50))
    m.load_state_dict({k: v for k, v in sd.items() if k in m.state_dict()}, strict=False)
    missing = {n for n, _ in m.named_parameters()} - set(sd)
    assert not missing, sorted(missing)
    return m.finalize_(torch.device(dev))


def site_seed_table(layer_type, layers, pre="encoder."):
    """{oracle site name: (layer, op)} for every dropout site of the encoder."""
    per = CONFORMER_SEEDS if layer_type == "conformer" else TRANSFORMER_SEEDS
    tab = {pre + k: v for k, v in ENCODER_SEEDS.items()}
    for li in range(layers):
        for role, (_, op) in per.items():
            tab[pre + "layers.%d.%s" % (li, role)] = (li, op)
    return tab


def engine_mask_provider(engine, layer_type, p, device_seed=0, seeds=None):
    """masks(site, x) for oracle/conformer.py: the fp32 multiplier keep * scale(p) the engine applied at that site.
    Activations are batch-major [B, T, C] with index (b * T + t) * C + c; attention probabilities [B, H, T, T] use the
    kernels' index ((h * B + b) * T + i) * ld + j with ld the padded probability stride."""
    seeds = site_seed_table(layer_type, engine.cfg["layers"]) if seeds is None else seeds
    sc = RNG.scale(p)
    seen = set()

    def masks(site, x):
        layer, op = seeds[site]
        seen.add(site)
        seed = RNG.combine_seed(engine._seed(layer, op), device_seed)
        if site.endswith("attn.probs"):
            B, H, T, _ = x.shape
            ld = (T + 7) // 8 * 8
            idx = torch.arange(H * B * T * ld, dtype=torch.int64).view(H, B, T, ld)[..., :T].permute(1, 0, 2, 3)
        else:
            idx = torch.arange(x.numel(), dtype=torch.int64).view(x.shape)
        return RNG.keep_mask(seed, idx, p).float() * sc

    masks.seen = seen
    return masks


def run_engine(m, g, dev):
    """One training forward + hand-written backward; returns (loss, logits [B, T', V] fp32 cpu, {name: grad})."""
    from espresso_b200.criterions import CtcLossCriterion

    crit = CtcLossCriterion(_Task(50))
    sample = {"net_input": {"src_tokens": torch.from_numpy(g["feats"]).to(dev), "src_lengths": torch.from_numpy(g["lens"]).to(dev)},
              "target": torch.from_numpy(g["target"]).to(dev), "ntokens": 13}
    got = {}
    fwd = m.forward

    def capture(*a, **kw):
        out = fwd(*a, **kw)
        got["logits"] = out["encoder_out"][0].transpose(0, 1).detach().float().cpu()
        return out

    m.forward = capture
    try:
        m.train()
        m.flat.zero_grad()
        loss, _, _ = crit(m, sample)
        loss.backward()
    finally:
        del m.forward
    m.encoder.sync_torch_grads_()
    names = [n for n, q in m.named_parameters() if n.startswith("encoder.")]
    grads = {n: m.flat.grad(n).detach().float().cpu().clone() for n in names}
    return float(loss.item()), got["logits"], grads


def run_oracle(sd0, g, layer_type, p, masks, d=64, H=4):
    """fp32 oracle training step on the bf16-rounded parameters the engine holds, masks injected at every site."""
    sd = {}
    for k, v in sd0.items():
        v = v.clone()
        if v.is_floating_point() and "running_" not in k:
            v = v.to(torch.bfloat16).float().requires_grad_(True)
        sd[k] = v
    cfg = dict(embed_dim=d, ffn_dim=128, heads=H, layers=2, layer_type=layer_type, dw_kernel=31, dropout=p,
               attention_dropout=p, activation_dropout=p, layernorm_embedding=True,
               final_layer_norm=layer_type != "conformer", vocab=50, dropout_masks=masks)
    logits, ol, _ = OC.encoder_forward(sd, cfg, torch.from_numpy(g["feats"]), torch.from_numpy(g["lens"]), training=True)
    loss = OC.ctc_criterion(logits, ol, torch.from_numpy(g["target"]), 1, 2, 0)
    loss.backward()
    grads = {k: v.grad for k, v in sd.items() if v.requires_grad and v.grad is not None}
    return float(loss.item()), logits.detach(), grads


def compare(layer_type, eng, orc):
    """-> dict of the errors: loss (relative), logits (max abs / max |ref|), per-tensor gradient rel-Frobenius."""
    (l_e, lg_e, g_e), (l_o, lg_o, g_o) = eng, orc
    worst = []
    for name, ge in g_e.items():
        if ("pre_encoder.convolutions" in name and name.endswith(".bias")) or name.endswith("k_proj.bias"):
            continue  # analytically zero gradients (bias feeding BatchNorm; key bias under softmax): rounding noise only
        go = g_o[name].reshape(ge.shape)
        worst.append((float(torch.linalg.norm(ge - go) / max(float(torch.linalg.norm(go)), 1e-3)), name))
    worst.sort(reverse=True)
    return dict(loss=abs(l_e - l_o) / abs(l_o), logits=float((lg_e - lg_o).abs().max() / lg_o.abs().max()), worst=worst,
                worst_body=max(w for w, n in worst if "pre_encoder" not in n), median=float(np.median([w for w, _ in worst])))
