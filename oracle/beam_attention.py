"""Oracle: the encoder attention of the beam search (`print_alignment`).  TEST INFRASTRUCTURE ONLY.

1. The two new ops of espresso_b200/ops.py restated in plain PyTorch, same signatures (fp32 arithmetic):
     decode_cross_attn_weights -- oracle/ops_ref.decode_cross_attn + the fp32 head-mean of the softmax probabilities
                                  (fairseq/modules/multihead_attention.py:864,913-915; padded keys exactly 0);
     beam_bookkeep_attn        -- oracle/ops_ref.beam_bookkeep + the attention columns att[t][anc[t][row]], t = 0..step, of
                                  every hypothesis it finalises (fairseq/sequence_generator.py:603-605,690,739-748).
   CPU tests monkeypatch them into `espresso_b200.ops` next to oracle/ops_ref.py.
2. Fp32EncDec: the encoder-decoder of tests/golden/encdec_transformer.npz in fp32 behind the generator protocol of
   espresso_b200/sequence_generator.py, recomputing the whole prefix every step (oracle/conformer.py encoder, the
   decoder of oracle/decoder.py) and recording the last layer's head-averaged encoder attention
   (fairseq/models/transformer/transformer_decoder.py:283-284).  It lets the host generator run with fp32 attention on the
   CPU; oracle/pin_beam_attention.py checks it against the real reference generator.
"""
import math

import torch
import torch.nn.functional as F

from oracle import conformer as OC
from oracle import ops_ref

ENC_CFG = dict(embed_dim=64, ffn_dim=128, heads=4, layers=2, layer_type="transformer", dropout=0.0, attention_dropout=0.0,
               activation_dropout=0.0, layernorm_embedding=False, final_layer_norm=True, vocab=None)
DEC_CFG = dict(dec_embed_dim=64, dec_heads=4, dec_layers=2, pad=1, max_target_positions=200)
PERTURB_SEED, PERTURB_SCALE = 31, 0.05
# The search fixture's model is the encdec fixture's with (1) the encoder-attention queries of decoder layer i scaled by
# Q_SCALE[i], so that the attention is peaked (the random-init model attends almost uniformly, which would hide a wrong
# row, step or layer) and differs between the layers, and (2) EOS_BIAS added to the eos logit through the final layer
# norm's bias direction, so that hypotheses end at different steps instead of all at max_len.
Q_SCALE = (40.0, 80.0)
EOS_BIAS = 0.75


def search_model(sd, eos=2):
    out = {k: torch.as_tensor(v).float().clone() for k, v in sd.items()}
    for i, a in enumerate(Q_SCALE):
        for kind in ("weight", "bias"):
            out["decoder.layers.%d.encoder_attn.q_proj.%s" % (i, kind)] *= a
    beta = out["decoder.layer_norm.bias"]
    out["decoder.output_projection.weight"][eos] += EOS_BIAS * beta / beta.dot(beta)
    return {k: v.numpy() for k, v in out.items()}


def perturbed(sd):
    """The second member of the fixture's ensemble: every tensor + PERTURB_SCALE * its std * N(0, 1) (seeded, CPU)."""
    g = torch.Generator().manual_seed(PERTURB_SEED)
    out = {}
    for k in sorted(sd):
        v = torch.as_tensor(sd[k]).float()
        noise = torch.randn(v.shape, generator=g)
        out[k] = (v + PERTURB_SCALE * (v.std() if v.numel() > 1 else v.abs()) * noise).numpy()
    return out


# ---- 1. ops --------------------------------------------------------------------------------------------------------
def decode_cross_attn_weights(q, kv, lens, beam, H, scale, weights):
    N, d = q.shape
    hd = d // H
    Tk = kv.shape[1]
    sent = torch.arange(N) // beam
    k = kv.float()[sent][..., :d].reshape(N, Tk, H, hd)
    s = torch.einsum("nhc,nthc->nht", q.float().reshape(N, H, hd), k) * scale
    if lens is not None:
        s = s.masked_fill((torch.arange(Tk)[None, :] >= lens.long()[sent][:, None])[:, None, :], float("-inf"))
    weights.copy_(torch.softmax(s, dim=-1).mean(dim=1))
    return ops_ref.decode_cross_attn(q, kv, lens, beam, H, scale)


def beam_bookkeep_attn(step, max_len, bsz, beam, K, eos, pad, normalize, len_penalty, cs, ct, cb, st, att, anc):
    fin = []  # (sentence, slot, source row): the finalisations beam_bookkeep is about to make, in its order
    for s in range(bsz):
        if st.finished[s]:
            continue
        slot = int(st.nfin[s])
        for c in range(min(beam, K)):
            if int(ct[s, c]) == eos and float(cs[s, c]) != float("-inf") and not st.ignore[s * beam + c] and slot < beam:
                fin.append((s, slot, s * beam + int(cb[s, c])))
                slot += 1
    ops_ref.beam_bookkeep(step, max_len, bsz, beam, K, eos, pad, normalize, len_penalty, cs, ct, cb, st)
    t = torch.arange(step + 1)
    for s, k, row in fin:
        st.fin_attn[s, k, : step + 1] = att[t, anc[: step + 1, row].long()]


# ---- 2. fp32 model ---------------------------------------------------------------------------------------------------
def decoder_step(sd, prefix, enc, enc_pad, cfg=DEC_CFG, pre="decoder."):
    """prefix [N, U] (no pad), enc [N, T', d], enc_pad bool [N, T'] -> (logits [N, V] of the last position, attention
    [N, T'] of the last layer at the last position, averaged over heads)."""
    pad, d, H = cfg["pad"], cfg["dec_embed_dim"], cfg["dec_heads"]
    N, U = prefix.shape
    hd = d // H
    half = d // 2
    f = torch.exp(torch.arange(half, dtype=torch.float) * -(math.log(10000) / (half - 1)))
    pos = torch.arange(pad + 1, pad + 1 + U, dtype=torch.float)[:, None] * f[None, :]
    x = math.sqrt(d) * F.embedding(prefix, sd[pre + "embed_tokens.weight"]) + torch.cat([torch.sin(pos), torch.cos(pos)], 1)

    def heads(t, w, b):
        return F.linear(t, w, b).view(N, t.shape[1], H, hd).transpose(1, 2)

    attn = None
    for i in range(cfg["dec_layers"]):
        p = pre + "layers.%d." % i
        for kind, causal in (("self_attn", True), ("encoder_attn", False)):
            ln = "self_attn_layer_norm" if causal else "encoder_attn_layer_norm"
            h = F.layer_norm(x, (d,), sd[p + ln + ".weight"], sd[p + ln + ".bias"])
            src = h if causal else enc
            q = heads(h, sd[p + kind + ".q_proj.weight"], sd[p + kind + ".q_proj.bias"]) * hd ** -0.5
            k = heads(src, sd[p + kind + ".k_proj.weight"], sd[p + kind + ".k_proj.bias"])
            v = heads(src, sd[p + kind + ".v_proj.weight"], sd[p + kind + ".v_proj.bias"])
            w = q @ k.transpose(-1, -2)
            if causal:
                w = w + torch.triu(torch.full((U, U), float("-inf")), 1)
            elif enc_pad is not None:
                w = w.masked_fill(enc_pad[:, None, None, :], float("-inf"))
            w = torch.softmax(w, dim=-1)
            if not causal:
                attn = w[:, :, -1].mean(dim=1)
            ctx = (w @ v).transpose(1, 2).reshape(N, U, d)
            x = x + F.linear(ctx, sd[p + kind + ".out_proj.weight"], sd[p + kind + ".out_proj.bias"])
        h = F.layer_norm(x, (d,), sd[p + "final_layer_norm.weight"], sd[p + "final_layer_norm.bias"])
        x = x + F.linear(F.relu(F.linear(h, sd[p + "fc1.weight"], sd[p + "fc1.bias"])), sd[p + "fc2.weight"], sd[p + "fc2.bias"])
    x = F.layer_norm(x[:, -1], (d,), sd[pre + "layer_norm.weight"], sd[pre + "layer_norm.bias"])
    return F.linear(x, sd[pre + "output_projection.weight"]), attn


class Fp32EncDec:
    """Generator-protocol model (see espresso_b200/sequence_generator.py) over a reference state_dict, fp32, on the CPU."""

    def __init__(self, sd):
        self.sd = {k: torch.as_tensor(v).float() for k, v in sd.items()}

    def max_decoder_positions(self):
        return DEC_CFG["max_target_positions"]

    def forward_encoder(self, net_input):
        with torch.no_grad():
            enc, _, pad = OC.encoder_forward(self.sd, ENC_CFG, net_input["src_tokens"].float(), net_input["src_lengths"])
        return {"enc": enc, "pad": pad if bool(pad.any()) else None}

    def init_incremental_state(self, enc, bsz, beam, attention=False):
        N, Tk = bsz * beam, enc["enc"].shape[1]
        T = self.max_decoder_positions() + 2
        return {"enc": enc, "beam": beam, "anc": torch.zeros(T, N, dtype=torch.int32), "anc_alt": torch.zeros(T, N, dtype=torch.int32),
                "attn": torch.zeros(T, N, Tk) if attention else None}

    def decode_step(self, step, tokens, state, new_order):
        ops_ref.decode_update_ancestry(state["anc"], state["anc_alt"], new_order if step > 0 else None, step)
        state["anc"], state["anc_alt"] = state["anc_alt"], state["anc"]
        sent = torch.arange(tokens.shape[0]) // state["beam"]
        e = state["enc"]
        with torch.no_grad():
            logits, attn = decoder_step(self.sd, tokens[:, : step + 1].long(), e["enc"][sent],
                                        None if e["pad"] is None else e["pad"][sent])
        if state["attn"] is not None:
            state["attn"][step] = attn
        return logits, True

    @staticmethod
    def decode_attention(state):
        return None if state["attn"] is None else (state["attn"], state["anc"])
