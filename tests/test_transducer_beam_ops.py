"""CPU: the plain-PyTorch statements of the transducer beam kernels (oracle/transducer_beam_ops.py), composed by
BatchedAdaptiveExpansionSearch, give every utterance of a batch exactly the n-best AdaptiveExpansionSearch gives it
alone, with the fp32 oracle model of oracle/transducer.py behind both (tests/golden/transducer_greedy.npz cases)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ops_ref, transducer_beam_ops

_CASES = [("beam5", dict(beam_size=5, max_num_expansions_per_step=3, expansion_beta=2, expansion_gamma=2.3, prefix_alpha=1,
                         temperature=1.3), False),
          ("beam3_lm", dict(beam_size=3, max_num_expansions_per_step=2, expansion_beta=1, expansion_gamma=4.0, prefix_alpha=2,
                            temperature=1.0), True),
          ("beam4_eos_a3", dict(beam_size=4, max_num_expansions_per_step=2, expansion_beta=0, expansion_gamma=None,
                                prefix_alpha=3, temperature=1.0, model_predicts_eos=True), False),
          ("beam1", dict(beam_size=1, max_num_expansions_per_step=2, expansion_beta=0, expansion_gamma=None, prefix_alpha=1,
                         temperature=1.0), False)]


@pytest.fixture()
def ref_ops(monkeypatch):
    from espresso_b200 import ops

    for mod in (ops_ref, transducer_beam_ops):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                monkeypatch.setattr(ops, name, getattr(mod, name))


def _fixture(golden_dir):
    from oracle import conformer as OC

    g = np.load(os.path.join(golden_dir, "transducer_conformer.npz"))
    gg = np.load(os.path.join(golden_dir, "transducer_greedy.npz"))
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    lm_sd = {k[len("lm.sd."):]: torch.from_numpy(gg[k]) for k in gg.files if k.startswith("lm.sd.")}
    ecfg = dict(embed_dim=64, ffn_dim=128, heads=4, layers=2, layer_type="conformer", dw_kernel=31, dropout=0.0,
                attention_dropout=0.0, activation_dropout=0.0, layernorm_embedding=True, final_layer_norm=False, vocab=None)
    with torch.no_grad():
        enc, ol, _ = OC.encoder_forward(sd, ecfg, torch.from_numpy(g["feats"]), torch.from_numpy(g["lens"]), training=False)
    return sd, lm_sd, enc, ol, gg


def batched_callbacks(sd, enc, lm_sd=None, n_layers=2, pad=1):
    """oracle.transducer.search_callbacks over a batch: the predictor output is its own "projection" and the joint takes
    the encoder frame of each row's utterance (frame = b * T + t)."""
    from oracle import transducer as OT

    T = enc.size(1)
    flat = enc.reshape(-1, enc.size(-1))
    cb = OT.search_callbacks(sd, enc[0], n_layers, pad, lm_sd=lm_sd)
    out = dict(pred_step=cb["pred_step"], init_state=cb["init_state"], project=lambda o: o,
               joint_logits=lambda frame, o: OT.joint_logits(sd, flat[frame.long()][:, None], o[:, None])[:, 0, 0])
    if lm_sd is not None:
        def lm_logits(feat):
            x = feat
            if "decoder.additional_fc.weight" in lm_sd:
                x = F.linear(x, lm_sd["decoder.additional_fc.weight"], lm_sd["decoder.additional_fc.bias"])
            w = lm_sd["decoder.fc_out.weight"] if "decoder.fc_out.weight" in lm_sd else lm_sd["decoder.embed_tokens.weight"]
            return F.linear(x, w, lm_sd.get("decoder.fc_out.bias") if "decoder.fc_out.weight" in lm_sd else None)

        out.update(lm_step=cb["lm_step"], lm_init_state=cb["lm_init_state"], lm_logits=lm_logits)
    assert T > 0
    return out


def _core(kw):
    from espresso_b200.tools.transducer_beam_search_decoder import AdaptiveExpansionSearch

    return AdaptiveExpansionSearch(50, 0, 1, 2, 2, kw["beam_size"], kw["max_num_expansions_per_step"], kw["expansion_beta"],
                                   kw["expansion_gamma"], kw["prefix_alpha"], True, kw.get("model_predicts_eos", False), 0.3, False)


def _host(core, sd, lm_sd, enc_b, n, kw, use_lm):
    from oracle import transducer as OT

    cb = OT.search_callbacks(sd, enc_b, 2, 1, temperature=kw["temperature"], lm_sd=lm_sd if use_lm else None)
    return core.search(n, cb, torch.device("cpu"), use_lm=use_lm)


def _assert_same(got, want):
    assert np.array_equal(got[0].numpy(), want[0].numpy()), (got[0], want[0])
    assert np.abs(got[1].numpy() - want[1].numpy()).max() < 1e-5


@pytest.mark.parametrize("name,kw,use_lm", _CASES)
def test_batched_statements_match_host_search(name, kw, use_lm, golden_dir, ref_ops):
    from espresso_b200.tools.transducer_beam_search_decoder import BatchedAdaptiveExpansionSearch

    sd, lm_sd, enc, ol, gg = _fixture(golden_dir)
    core = _core(kw)
    search = BatchedAdaptiveExpansionSearch(core, kw["temperature"])
    with torch.no_grad():
        got = search.search(ol.int(), enc.size(1), batched_callbacks(sd, enc, lm_sd if use_lm else None), torch.device("cpu"),
                            use_lm=use_lm)
        for b in range(enc.size(0)):
            want = _host(core, sd, lm_sd, enc[b], int(ol[b]), kw, use_lm)
            _assert_same(got[b], want)
            if name + "_b0_seqs" in gg.files:
                assert np.array_equal(got[b][0].numpy(), gg["%s_b%d_seqs" % (name, b)])


@pytest.mark.parametrize("name,kw,use_lm", _CASES[:2])
def test_batch_of_cut_utterances_matches_each_alone(name, kw, use_lm, golden_dir, ref_ops):
    """Utterances cut to different frame counts in one batch: each gets the n-best it gets searched alone, and an
    utterance whose frames end early is left untouched while the others go on."""
    from espresso_b200.tools.transducer_beam_search_decoder import BatchedAdaptiveExpansionSearch

    sd, lm_sd, enc, ol, _ = _fixture(golden_dir)
    cuts = torch.tensor([int(ol[0]), max(int(ol[1]) // 3, 1), 0 if int(ol[2]) < 2 else int(ol[2]) - 1, int(ol[0]) // 2], dtype=torch.int32)
    batch = torch.cat([enc, enc[:1]], 0)
    core = _core(kw)
    with torch.no_grad():
        got = BatchedAdaptiveExpansionSearch(core, kw["temperature"]).search(
            cuts, batch.size(1), batched_callbacks(sd, batch, lm_sd if use_lm else None), torch.device("cpu"), use_lm=use_lm)
        for b in range(batch.size(0)):
            if int(cuts[b]) == 0:
                continue
            _assert_same(got[b], _host(core, sd, lm_sd, batch[b], int(cuts[b]), kw, use_lm))
