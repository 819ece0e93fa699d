"""Pin oracle/abspos.py against the REAL reference and write tests/golden/{encdec_transformer_abspos,
encdec_transformer_abspos_hd128,encoder_conformer_abspos}.npz.

Runs only where the reference tree is available (imported through oracle/refshim):
    python -m oracle.pin_abspos
Models with relative positions OFF (the WSJ / Switchboard Transformer recipes' setting: examples/asr_wsj/run.sh,
examples/asr_swbd/run.sh, speech_transformer_legacy.py:125-127): two encoder-decoder models shaped like the WSJ recipe
(head dim 64, relaxed encoder attention 0.35, temporal smoothing 0.05) and the Switchboard recipe (head dim 128, uniform
smoothing 0.1), and a Conformer + CTC encoder.  Parameters come from oracle.abspos.seeded_state_dict (not stored).
Training mode at dropout 0 (relaxation is active in training only): logits, loss, nll and a sketch of every gradient;
eval-mode logits afterwards (relaxation off; BatchNorm running statistics as the training forward left them, stored);
the reference's state-dict keys.  The oracle must reproduce the reference before anything is written."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

from oracle import abspos as O
from oracle import refshim

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
V, PAD, EOS, BLANK = 50, 1, 2, 0
SD_SEED = 1


def _cfg(layer_type, d, ffn, heads, layers, relaxed=0.0):
    from espresso.models.transformer.speech_transformer_config import SpeechTransformerConfig

    cfg = SpeechTransformerConfig()
    cfg.max_source_positions, cfg.max_target_positions, cfg.tpu = 3600, 200, False
    e = cfg.encoder
    e.conv_channels = "[64, 64, 128, 128]"
    e.conv_kernel_sizes = "[(3, 3), (3, 3), (3, 3), (3, 3)]"
    e.conv_strides = "[(1, 1), (2, 2), (1, 1), (2, 2)]"
    e.embed_dim, e.ffn_embed_dim, e.layers, e.attention_heads = d, ffn, layers, heads
    e.normalize_before, e.learned_pos, e.relative_positional_embeddings = True, False, False
    e.layer_type, e.depthwise_conv_kernel_size = layer_type, 31
    dc = cfg.decoder
    dc.embed_dim, dc.ffn_embed_dim, dc.layers, dc.attention_heads = d, ffn, layers, heads
    dc.normalize_before, dc.learned_pos, dc.relative_positional_embeddings = True, False, False
    dc.input_dim, dc.output_dim = d, d
    dc.relaxed_attention_weight = relaxed
    cfg.dropout = cfg.attention_dropout = cfg.activation_dropout = 0.0
    return cfg


class _Dict:
    def __len__(self):
        return V

    def pad(self):
        return PAD

    def eos(self):
        return EOS


class _Task:
    feat_dim, feat_in_channels, target_dictionary = 80, 1, _Dict()


def inputs(seed, U):
    rs = np.random.RandomState(seed)
    B, T = 3, 61
    lens = torch.tensor([61, 50, 37])
    feats = torch.from_numpy(rs.randn(B, T, 80).astype(np.float32))
    for b in range(B):
        feats[b, lens[b]:] = 0.0
    tgt = torch.full((B, U), PAD, dtype=torch.long)
    prev = torch.full((B, U), PAD, dtype=torch.long)
    for b, u in enumerate((U - 1, U - 3, U - 5)):
        toks = torch.from_numpy(rs.randint(4, V, size=u))
        tgt[b, :u] = toks
        tgt[b, u] = EOS
        prev[b, 0] = EOS
        prev[b, 1:u + 1] = toks
    return feats, lens, tgt, prev


def _seed_params(m):
    sd = O.seeded_state_dict({k: v.shape for k, v in m.state_dict().items()}, SD_SEED)
    torch.nn.Module.load_state_dict(m, sd, strict=True)  # plain load: fairseq's upgrade hooks do not apply here
    return {k: v.clone() for k, v in m.state_dict().items()}


def _oracle_sd(sd0, m):
    pnames = dict(m.named_parameters())
    return {k: v.clone().requires_grad_(k in pnames) for k, v in sd0.items()}


def _check_grads(m, sd, out):
    worst = 0.0
    for n, p_ in m.named_parameters():
        out["gsk." + n] = O.grad_sketch(n, p_.grad)
        if O.skip_grad(n):
            continue
        dg = (sd[n].grad - p_.grad).norm().item() / max(p_.grad.norm().item(), 1e-3)
        worst = max(worst, dg)
    print("   worst relative gradient difference (Frobenius) %.3g" % worst)
    assert worst < 2e-4


def pin_encdec():
    from espresso.criterions.label_smoothed_cross_entropy_v2 import label_smoothed_nll_loss, temporal_label_smoothing_prob_mask
    from espresso.models.transformer.speech_transformer_base import SpeechTransformerModelBase

    for name, d, ffn, heads, L, relaxed, smoothing, eps in (
            ("encdec_transformer_abspos", 128, 256, 2, 2, 0.35, "temporal", 0.05),
            ("encdec_transformer_abspos_hd128", 256, 512, 2, 1, 0.0, "uniform", 0.1)):
        torch.manual_seed(3)
        m = SpeechTransformerModelBase.build_model(_cfg("transformer", d, ffn, heads, L, relaxed), _Task())
        sd0 = _seed_params(m)
        feats, lens, tgt, prev = inputs(13, 8)
        ecfg = dict(heads=heads, layers=L, layer_type="transformer", final_layer_norm=True, vocab=None)
        dcfg = dict(dec_embed_dim=d, dec_heads=heads, dec_layers=L, pad=PAD, relaxed_attention_weight=relaxed)
        out = {}
        m.train()
        m.zero_grad()
        logits, extra = m(feats, lens, prev)
        lprobs = m.get_normalized_probs((logits, extra), log_probs=True)
        mask = temporal_label_smoothing_prob_mask(lprobs, tgt, PAD) if smoothing == "temporal" else None
        loss, nll = label_smoothed_nll_loss(lprobs.view(-1, lprobs.size(-1)), tgt.view(-1), eps, ignore_index=PAD,
                                            reduce=True, smoothing_type=smoothing, prob_mask=mask)
        loss.backward()
        sd = _oracle_sd(sd0, m)
        enc, _, pad = O.encoder_forward(sd, ecfg, feats, lens, training=True)
        o_logits = O.decoder_forward(sd, dcfg, prev, enc, pad if bool(pad.any()) else None, training=True)
        o_loss, o_nll = O.smoothed_ce(o_logits, tgt, PAD, eps, smoothing, V)
        o_loss.backward()
        dl = (o_logits - logits).abs().max().item()
        print("%s: |logits diff|=%.3g loss ref=%.6f oracle=%.6f nll ref=%.6f oracle=%.6f" % (
            name, dl, loss.item(), o_loss.item(), nll.item(), o_nll.item()))
        assert dl < 2e-4 and abs(loss.item() - o_loss.item()) < 1e-4 * abs(loss.item())
        _check_grads(m, sd, out)
        out.update({"after." + k: v.numpy() for k, v in m.state_dict().items() if "running_" in k})
        out["logits"] = logits.detach().numpy()
        m.eval()
        with torch.no_grad():
            logits_eval, _ = m(feats, lens, prev)
            sd_after = {k: v.clone() for k, v in m.state_dict().items()}
            enc_e, _, pad_e = O.encoder_forward(sd_after, ecfg, feats, lens, training=False)
            o_eval = O.decoder_forward(sd_after, dcfg, prev, enc_e, pad_e if bool(pad_e.any()) else None, training=False)
        de = (o_eval - logits_eval).abs().max().item()
        print("   eval |logits diff|=%.3g" % de)
        assert de < 2e-4
        out.update(feats=feats.numpy(), lens=lens.numpy(), target=tgt.numpy(), prev_output_tokens=prev.numpy(),
                   logits_eval=logits_eval.numpy(), loss=np.float64(loss.item()), nll=np.float64(nll.item()),
                   eps=np.float64(eps), smoothing=np.array(smoothing), relaxed=np.float64(relaxed), sd_seed=np.int64(SD_SEED),
                   embed_dim=np.int64(d), ffn_dim=np.int64(ffn), heads=np.int64(heads), layers=np.int64(L),
                   state_dict_keys=np.array(sorted(m.state_dict().keys())))
        np.savez_compressed(os.path.join(GOLDEN, name + ".npz"), **out)
        print("%s pinned -> tests/golden/%s.npz" % (name, name))


def pin_conformer():
    from espresso.models.transformer.speech_transformer_encoder_model import SpeechTransformerEncoderModel

    from oracle import conformer as OC

    d, ffn, heads, L = 128, 256, 2, 2
    cfg = _cfg("conformer", d, ffn, heads, L)
    cfg.layernorm_embedding = True
    torch.manual_seed(1)
    m = SpeechTransformerEncoderModel.build_model(cfg, _Task())
    _seed_params(m)
    feats, lens, tgt, _ = inputs(11, 7)
    ecfg = dict(heads=heads, layers=L, layer_type="conformer", layernorm_embedding=True, final_layer_norm=False, vocab=V)
    out = {}
    for mode in ("train", "eval"):
        m.train(mode == "train")
        sd0 = {k: v.clone() for k, v in m.state_dict().items()}
        m.zero_grad()
        net = m(feats, lens)
        logits = net["encoder_out"][0]
        olens = net["src_lengths"][0]
        lprobs = m.get_normalized_probs(net, log_probs=True).contiguous()
        keep = (tgt != PAD) & (tgt != EOS)
        loss = F.ctc_loss(lprobs, tgt.masked_select(keep), olens, keep.sum(-1), blank=BLANK, reduction="sum", zero_infinity=True)
        sd = _oracle_sd(sd0, m)
        o_logits, o_lens, _ = O.encoder_forward(sd, ecfg, feats, lens, training=(mode == "train"))
        o_loss = OC.ctc_criterion(o_logits, o_lens, tgt, PAD, EOS, BLANK)
        d_log = (o_logits.transpose(0, 1) - logits).abs().max().item()
        assert torch.equal(o_lens, olens)
        print("conformer_abspos/%s: |logits diff|=%.3g loss ref=%.6f oracle=%.6f" % (mode, d_log, loss.item(), o_loss.item()))
        assert d_log < 2e-4 and abs(o_loss.item() - loss.item()) < 1e-4 * abs(loss.item())
        if mode == "train":
            loss.backward()
            o_loss.backward()
            _check_grads(m, sd, out)
            out.update({"after." + k: v.numpy() for k, v in m.state_dict().items() if "running_" in k})
        out["logits_" + mode] = logits.detach().transpose(0, 1).numpy()
        out["loss_" + mode] = np.float64(loss.item())
    out.update(feats=feats.numpy(), lens=lens.numpy(), target=tgt.numpy(), out_lens=olens.numpy(), sd_seed=np.int64(SD_SEED),
               embed_dim=np.int64(d), ffn_dim=np.int64(ffn), heads=np.int64(heads), layers=np.int64(L),
               state_dict_keys=np.array(sorted(m.state_dict().keys())))
    np.savez_compressed(os.path.join(GOLDEN, "encoder_conformer_abspos.npz"), **out)
    print("conformer abspos encoder pinned -> tests/golden/encoder_conformer_abspos.npz")


def main(argv):
    refshim.activate()
    for name in (argv or ["encdec", "conformer"]):
        {"encdec": pin_encdec, "conformer": pin_conformer}[name]()


if __name__ == "__main__":
    main(sys.argv[1:])
