"""Pin the beam search's encoder attention (`print_alignment`) against the REAL reference and write
tests/golden/beam_attention.npz.

Runs only where the reference tree is present (imported through oracle/refshim):
    python -m oracle.pin_beam_attention
The reference SequenceGenerator (fairseq/sequence_generator.py, Espresso's version) decodes in fp32, eval mode, with the
reference SpeechTransformerModelBase holding the weights of tests/golden/encdec_transformer.npz, on that fixture's ragged
utterances, with the decoder's encoder-attention queries sharpened and an eos bias (oracle.beam_attention.search_model):
beam 4 with the full n-best; a two-model ensemble (that model plus a seeded perturbed copy); and a max_len that forces eos.
Hypotheses end at several steps, some with a natural eos, some at max_len.  The same cases are then decoded by espresso_b200.SequenceGenerator on the CPU with
oracle/ops_ref.py + oracle/beam_attention.py patched in for the native ops and oracle.beam_attention.Fp32EncDec as the
model(s): tokens must be identical and every attention matrix within 1e-5.  The fixture stores the inputs, checksums of the two
models' weights (oracle.beam_attention regenerates them), per case / sentence / hypothesis the tokens, scores and
[T', len(tokens)] attention, and per sentence its decision margin: the smallest gap between adjacent scores among the best
2 * beam + 1 candidates over the steps of its search.  A search whose score errors stay below half of it takes the same
decisions, so it finds the same n-best.
"""
import argparse
import os

import numpy as np
import torch

from oracle import refshim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = [  # name, models, generator arguments
    ("beam4", 1, dict(beam_size=4, max_len_a=0.0, max_len_b=40)),
    ("ensemble", 2, dict(beam_size=4, max_len_a=0.0, max_len_b=40)),
    ("maxlen", 1, dict(beam_size=4, max_len_a=0.0, max_len_b=3)),
]
class _Dict:
    def __init__(self, V):
        self.V = V

    def __len__(self):
        return self.V

    def pad(self):
        return 1

    def eos(self):
        return 2

    def unk(self):
        return 3

    def bos(self):
        return 0


def reference_model(sd, V):
    from espresso.models.transformer.speech_transformer_base import SpeechTransformerModelBase
    from espresso.models.transformer.speech_transformer_config import SpeechTransformerConfig

    cfg = SpeechTransformerConfig()
    cfg.max_source_positions, cfg.max_target_positions, cfg.tpu = 3600, 200, False
    e = cfg.encoder
    e.conv_channels = "[64, 64, 128, 128]"
    e.conv_kernel_sizes = "[(3, 3), (3, 3), (3, 3), (3, 3)]"
    e.conv_strides = "[(1, 1), (2, 2), (1, 1), (2, 2)]"
    e.embed_dim, e.ffn_embed_dim, e.layers, e.attention_heads = 64, 128, 2, 4
    e.normalize_before, e.learned_pos, e.relative_positional_embeddings, e.layer_type = True, False, True, "transformer"
    d = cfg.decoder
    d.embed_dim, d.ffn_embed_dim, d.layers, d.attention_heads = 64, 128, 2, 4
    d.normalize_before, d.learned_pos, d.relative_positional_embeddings = True, False, False
    d.input_dim, d.output_dim = 64, 64
    cfg.dropout = cfg.attention_dropout = cfg.activation_dropout = 0.0

    class _Task:
        feat_dim, feat_in_channels, target_dictionary = 80, 1, _Dict(V)

    m = SpeechTransformerModelBase.build_model(cfg, _Task())
    m.load_state_dict({k: torch.as_tensor(v) for k, v in sd.items()}, strict=True)
    return m.float().eval()


def product_generate(sds, V, feats, lens, kw, gaps=None):
    """espresso_b200.SequenceGenerator on the CPU over the oracle ops and fp32 models (what tests/test_beam_attention.py runs).
    gaps: a list that receives, per search step, [bsz] the smaller of each sentence's two cut gaps: between its beam-th and
    (beam+1)-th best candidate, and between the 2*beam-th and (2*beam+1)-th (what enters the top-k)."""
    from espresso_b200 import ops
    from espresso_b200.sequence_generator import SequenceGenerator
    from oracle import beam_attention as OA
    from oracle import ops_ref

    saved = {}
    for mod in (ops_ref, OA):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                saved.setdefault(name, getattr(ops, name))
                setattr(ops, name, getattr(mod, name))

    def topk(cand, bsz, sent_stride, n_cand, K, V_):
        c = cand.reshape(-1)[: bsz * sent_stride].view(bsz, sent_stride)[:, :n_cand]
        top = c.topk(min(K + 1, n_cand), dim=1).values
        nb = min(K // 2, top.shape[1] - 1)  # beam
        gap = torch.stack([top[:, nb - 1] - top[:, nb], top[:, -2] - top[:, -1]], dim=1)
        gaps.append(torch.where(torch.isfinite(gap), gap, torch.full_like(gap, float("inf"))).min(dim=1).values)
        return ops_ref.beam_topk(cand, bsz, sent_stride, n_cand, K, V_)

    if gaps is not None:
        ops.beam_topk = topk
    try:
        models = [OA.Fp32EncDec(sd) for sd in sds]
        gen = SequenceGenerator(models, _Dict(V), print_alignment=True, **kw)
        return gen.generate(models, {"net_input": {"src_tokens": feats, "src_lengths": lens}})
    finally:
        for name, fn in saved.items():
            setattr(ops, name, fn)


def main(argv=None):
    argparse.ArgumentParser(description=__doc__.splitlines()[0]).parse_args(argv)
    refshim.activate()
    from fairseq.sequence_generator import SequenceGenerator

    from oracle import beam_attention as OA

    g = np.load(os.path.join(GOLDEN, "encdec_transformer.npz"))
    sd1 = OA.search_model({k[3:]: g[k] for k in g.files if k.startswith("sd.")})
    sd2 = OA.perturbed(sd1)
    V = 50
    feats, lens = torch.from_numpy(g["feats"]), torch.from_numpy(g["lens"])
    out = {"feats": g["feats"], "lens": g["lens"], "V": np.int64(V)}
    out["sd1_abs_sum"] = np.float64(sum(np.abs(v).astype(np.float64).sum() for v in sd1.values()))
    out["sd2_abs_sum"] = np.float64(sum(np.abs(v).astype(np.float64).sum() for v in sd2.values()))
    worst = 0.0
    for name, n_models, kw in CASES:
        sds = [sd1, sd2][:n_models]
        ref_models = [reference_model(sd, V) for sd in sds]
        gen = SequenceGenerator(ref_models, _Dict(V), **kw)
        with torch.no_grad():
            ref = gen.forward({"net_input": {"src_tokens": feats, "src_lengths": lens}})
        gaps = []
        ours = product_generate(sds, V, feats, lens, kw, gaps)
        for b, (rh, oh) in enumerate(zip(ref, ours)):
            assert len(rh) == len(oh), (name, b, len(rh), len(oh))
            for k, (r_, o_) in enumerate(zip(rh, oh)):
                assert r_["tokens"].tolist() == o_["tokens"].tolist(), (name, b, k)
                ra = r_["attention"].float()
                assert ra.shape == o_["attention"].shape, (name, b, k, ra.shape, o_["attention"].shape)
                err = (ra - o_["attention"]).abs().max().item()
                worst = max(worst, err)
                assert err < 1e-5, (name, b, k, err)
                key = "%s_b%d_k%d_" % (name, b, k)
                out[key + "tokens"] = r_["tokens"].numpy()
                out[key + "score"] = np.float32(float(r_["score"]))
                out[key + "attention"] = ra.numpy()
            out["%s_b%d_n" % (name, b)] = np.int64(len(rh))
            last = max(len(h["tokens"]) for h in rh)  # the sentence's search ended at step last - 1
            out["%s_b%d_margin" % (name, b)] = np.float32(min(float(gs[b]) for gs in gaps[:last]))
        print("beam attention %-8s: hypothesis lengths %s, decision margins %s" % (
            name, [[len(h["tokens"]) for h in hs] for hs in ref], [round(float(out["%s_b%d_margin" % (name, b)]), 3) for b in range(len(ref))]))
    out["cases"] = np.array([c[0] for c in CASES])
    print("worst |attention - reference| of the host generator over the oracle: %.3g" % worst)
    np.savez_compressed(os.path.join(GOLDEN, "beam_attention.npz"), **out)
    print("beam attention pinned -> tests/golden/beam_attention.npz")


if __name__ == "__main__":
    main()
