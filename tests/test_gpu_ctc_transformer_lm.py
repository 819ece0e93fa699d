"""GPU: CTC prefix beam search fused with a Transformer LM over the frame-slot KV cache.
  1. esp_decode_update_paths against a host simulation of the path tables, integer-exact after every frame;
  2. the LM's prefix step (esp_decode_self_attn_paths + per-row positions) under random (new_order, grown, fed) against
     a teacher-forced forward of every row's prefix, in fp32 (oracle/decoder.py) and through the native DecoderEngine;
  3. the fused search against oracle/ctc_beam.py with the float64 teacher-forced LM (test_gpu_ctc_beam._compare);
  4. CTCDecoder.generate and recognize() end to end.
Every bound is recorded with the error reached through the `parity` fixture."""
import math
import os
from argparse import Namespace

import numpy as np
import pytest
import torch

import test_gpu_ctc_beam as G
from test_ctc_beam_search import _dict
from test_ctc_transformer_lm import LOGIT_ULPS, lm_oracle_fn, random_frames, simulate_paths, tlm, tlm_teacher_forced

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
# the LM runs in bf16 on the device and in float64 in the oracle: its log-probabilities differ by a few bf16 ulps of the
# logits (test 2), times lm_weight per emitted token.  Hypotheses whose oracle margin exceeds LM_MARGIN must match
# exactly; scores agree within LM_SCORE_TOL relative, twice the largest error reached on an H100 (4.8e-3, beam 16 with
# the blank left out of the LM; the errors reached are recorded next to the bound).
LM_MARGIN = 0.2
LM_SCORE_TOL = 1e-2


def _tables(N, T):
    z = lambda *s: torch.zeros(*s, dtype=torch.int32, device=DEV)  # noqa: E731
    return z(T + 1, N), z(N), z(T + 1, N), z(N), z(N)


# ---- 1. path tables --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bsz,beam", [(4, 16), (24, 60)])
@pytest.mark.parametrize("mode", ["random", "all_grow", "none_grow", "one_parent"])
def test_update_paths_exact(bsz, beam, mode):
    from espresso_b200 import ops

    N, T = bsz * beam, 40
    frames = random_frames(N, T, 50, seed=N + len(mode), mode=mode, beam=beam)
    hist = simulate_paths(frames, N, eos=2)
    cells, ln, c2, l2, pos = _tables(N, T)
    ix = torch.arange(N, dtype=torch.int32, device=DEV)
    steps = [(ix, torch.ones_like(ix))] + [(no.to(DEV), gr.to(DEV)) for no, gr, _ in frames]
    for slot, (no, gr) in enumerate(steps):
        ops.decode_update_paths(cells, ln, c2, l2, no, gr, slot, pos_out=pos)
        exp_pos = ln.cpu()[no.long().cpu()]
        cells, ln, c2, l2 = c2, l2, cells, ln
        got_c, got_l = cells.cpu().numpy(), ln.cpu().numpy()
        exp_l = np.array([len(c) for c, _ in hist[slot]])
        assert np.array_equal(got_l, exp_l), (mode, slot)
        assert torch.equal(pos.cpu(), exp_pos)
        exp_c = np.full_like(got_c, -1)
        for n, (c, _) in enumerate(hist[slot]):
            exp_c[: len(c), n] = c
        mask = np.arange(T + 1)[:, None] < exp_l[None, :]
        assert np.array_equal(np.where(mask, got_c, -1), exp_c), (mode, slot)
    if mode == "all_grow":
        assert (ln == T + 1).all()  # every row holds eos + T' tokens: all T' + 1 slots
    if mode == "none_grow":
        assert (ln == 1).all()


# ---- 2. the prefix step against teacher forcing ----------------------------------------------------------------------
@pytest.mark.parametrize("bsz,beam,lm_blank", [(4, 16, False), (2, 8, True)])
def test_prefix_step_vs_teacher_forcing(bsz, beam, lm_blank, parity):
    d = _dict(n_sym=36, bos=not lm_blank)
    lm = tlm(d, seed=3 + int(lm_blank), dim=64, layers=2, heads=4, device=DEV)
    V_lm = len(d)
    N, T = bsz * beam, 40
    tf32 = tlm_teacher_forced(lm, dtype=torch.float32)
    frames = random_frames(N, T, V_lm, seed=11 + int(lm_blank), beam=beam)
    hist = simulate_paths(frames, N, d.eos())
    st = lm.init_prefix_state(bsz, beam, T)
    ix = torch.arange(N, dtype=torch.int32, device=DEV)
    rows = lm.prefix_step(0, torch.full((N,), d.eos(), dtype=torch.int32, device=DEV), torch.ones_like(ix), ix, st)
    err_o, err_n, scale = 0.0, 0.0, 0.0
    for f in range(T + 1):
        if f > 0:
            no, gr, fed = (a.to(DEV) for a in frames[f - 1])
            new_rows = lm.prefix_step(f, fed, gr, no, st)
            rows = torch.where(gr.view(N, 1) != 0, new_rows, rows.index_select(0, no.long()))
        prefixes = [tk for _, tk in hist[f]]
        got = rows[:, :V_lm].float().cpu()
        scale = max(scale, float(got.abs().max()))
        err_o = max(err_o, float((torch.log_softmax(got.double(), -1) - tf32(prefixes).double()).abs().max()))
        # the native teacher-forced forward of the same prefixes, right-padded
        U = max(len(p) for p in prefixes)
        tok = torch.full((N, U), d.pad(), dtype=torch.int32)
        for i, p in enumerate(prefixes):
            tok[i, :len(p)] = torch.tensor(p, dtype=torch.int32)
        lens = torch.tensor([len(p) for p in prefixes], dtype=torch.int32)
        full = lm.engine.forward(tok.to(DEV), None, None, lens.to(DEV), save=False).float().cpu()
        ref = full[torch.arange(N), lens.long() - 1, :V_lm]
        err_n = max(err_n, float((got - ref).abs().max()))
    bound = LOGIT_ULPS * max(1.0, scale)
    parity("ctc prefix step N=%d lm_blank=%s vs fp32 teacher forcing: |log-softmax| abs err" % (N, lm_blank), err_o, bound)
    parity("ctc prefix step N=%d lm_blank=%s vs native teacher forcing: |logit| abs err" % (N, lm_blank), err_n, bound)


# ---- 3. the fused search against the oracle --------------------------------------------------------------------------
def _fixture_logits(golden_dir):
    from test_gpu_encoder import _build, _sample

    g = np.load(os.path.join(golden_dir, "encoder_conformer.npz"))
    m = _build("conformer", g)
    m.eval()
    sample = _sample(g, DEV)
    with torch.no_grad():
        net = m(**sample["net_input"])
    return m, sample, net["encoder_out"][0].size(-1), net["b200_out"].cpu(), net["src_lengths"][0].cpu()


@pytest.mark.parametrize("beam,lm_blank", [(4, False), (4, True), (16, False), (16, True), (60, False), (60, True)])
def test_search_transformer_lm_fusion(beam, lm_blank, golden_dir, parity, monkeypatch):
    _, _, V, x, lens = _fixture_logits(golden_dir)
    # the fixture's sentences plus two ragged ones: T' = 1 and T' = 0
    x = torch.cat([x, x[:1], x[:1]], 0)
    lens = torch.cat([lens, torch.tensor([1, 0], dtype=lens.dtype)])
    lm = tlm(_dict(n_sym=V - 4, bos=not lm_blank), seed=beam, dim=64, layers=2, heads=4, device=DEV)
    dec = G._decoder(V, beam, lm=lm, lm_weight=0.47, word_score=0.6, nbest=3, print_alignment=True)
    assert dec.transformer and dec.lm_blank == (0 if lm_blank else -1)
    lm_fn = lm_oracle_fn(lm, V, dec.eos, dec.lm_blank)
    monkeypatch.setattr(G, "MARGIN", LM_MARGIN)
    monkeypatch.setattr(G, "SCORE_TOL", LM_SCORE_TOL)
    G._compare(parity, "ctc beam + Transformer LM beam=%d lm_blank=%s" % (beam, lm_blank), dec, x, lens, V, lm_fn=lm_fn)


# ---- 4. end to end ---------------------------------------------------------------------------------------------------
def _peaked_lm(d, favourite, device):
    """A Transformer LM that predicts `favourite` after every context: final LayerNorm -> constant vector, output row
    of the favourite aligned with it."""
    from espresso_b200.models.transformer_lm import TransformerLanguageModel

    torch.manual_seed(0)
    lm = TransformerLanguageModel(d, embed_dim=64, ffn_embed_dim=128, layers=2, attention_heads=4,
                                  share_decoder_input_output_embed=False)
    with torch.no_grad():
        lm.decoder.layer_norm.weight.zero_()
        lm.decoder.layer_norm.bias.fill_(1.0)
        lm.decoder.output_projection.weight.zero_()
        lm.decoder.output_projection.weight[favourite] = 0.25
    return lm.finalize_(device).eval()


def test_generate_fixture_conformer_lm_weight_changes_hypotheses(golden_dir):
    m, sample, V, x, lens = _fixture_logits(golden_dir)
    fav = 7
    lm = _peaked_lm(_dict(n_sym=V - 4), fav, DEV)
    hyps = {}
    for w in (0.0, 3.0):
        dec = G._decoder(V, 8, lm=lm, lm_weight=w, nbest=2, print_alignment=True)
        hy = dec.generate([m], sample)
        assert len(hy) == x.shape[0]
        for b, hs in enumerate(hy):
            assert 1 <= len(hs) <= 2 and [h["score"] for h in hs] == sorted((h["score"] for h in hs), reverse=True)
            for h in hs:
                assert set(h) == {"tokens", "score", "attention", "alignment", "positional_scores"}
                t, a = h["tokens"], h["alignment"]
                assert t.dtype == torch.int64 and a.shape == t.shape and math.isfinite(h["score"])
                assert all(0 <= f < int(lens[b]) for f in a.tolist()) and a.tolist() == sorted(set(a.tolist()))
                assert not any(v in (0, 1, 2, 3) for v in t.tolist())
        hyps[w] = [hs[0]["tokens"].tolist() for hs in hy]
    assert hyps[0.0] != hyps[3.0]
    # every token but the favourite costs about lm_weight * 16 nats: the fused search emits fewer of them
    others = lambda hs: sum(len(h) - h.count(fav) for h in hs)  # noqa: E731
    assert others(hyps[3.0]) < others(hyps[0.0])


def test_recognize_ctc_with_transformer_lm_on_the_device(tmp_path):
    from test_input_pipeline import _corpus

    from espresso_b200.data.asr_dictionary import AsrDictionary
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel
    from espresso_b200.speech_recognize import recognize
    from espresso_b200.tasks.speech_recognition import SpeechRecognitionEspressoConfig, SpeechRecognitionEspressoTask

    d0, man = _corpus(tmp_path, n=5, fmt="wave")
    os.rename(str(tmp_path / "train.json"), str(tmp_path / "test.json"))
    d = AsrDictionary(enable_bos=True)
    for s in d0.symbols[d0.nspecial:]:
        d.add_symbol(s)
    d.space_index = d.index("<space>")
    d.build_bpe("characters_asr")
    task = SpeechRecognitionEspressoTask(SpeechRecognitionEspressoConfig(criterion_name="ctc_loss", data=str(tmp_path)), d,
                                         feat_dim=80)
    torch.manual_seed(4)
    mcfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, layernorm_embedding=False,
        encoder=dict(embed_dim=64, ffn_embed_dim=128, layers=1, attention_heads=4, normalize_before=True, learned_pos=False,
                     relative_positional_embeddings=True, layer_type="transformer")))
    m = SpeechTransformerEncoderModel.build_model(mcfg, task).finalize_(DEV)
    m.frontend = OnTheFlyFbank(None, None)
    lm = _peaked_lm(d, d.index("<space>"), DEV)
    run = lambda lms, w: recognize(task, [m], subset="test", gen_args=Namespace(beam=4, lm_weight=w), lms=lms,  # noqa: E731
                                   max_tokens=None, max_sentences=2, device="cuda:0")
    plain, fused = run(None, 0.0), run([lm], 3.0)
    hyp = lambda out: {l.split("\t")[0]: l.split("\t")[1] for l in out["lines"] if l.startswith("H-")}  # noqa: E731
    assert len(hyp(fused)) == len(man) and hyp(plain) != hyp(fused)
