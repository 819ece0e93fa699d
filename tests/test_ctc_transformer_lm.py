"""CPU: CTC prefix beam search fused with a Transformer LM.  The constructor's acceptance and refusals, build_generator /
recognize() routing, the path tables of the frame-slot KV cache, and the LM's prefix step run over oracle/ops_ref +
oracle/prefix_decode_ops against a float64 teacher-forced forward of the same LM (oracle/decoder.py) on eos + each
hypothesis's prefix, frame by frame under random (new_order, grown, fed)."""
import math
from argparse import Namespace

import numpy as np
import pytest
import torch

from test_ctc_beam_search import _FakeCTC, _dict, _logits, _task

# bf16 rounding of a logit of magnitude ~|x| is 2^-9 |x|; the engine rounds every activation, so allow a few ulps of the
# largest logit (the same bound the GPU test uses for the device kernels)
LOGIT_ULPS = 8 * 2.0 ** -8


def tlm(d, seed=0, dim=16, layers=2, heads=2, max_pos=1024, device=torch.device("cpu")):
    from espresso_b200.models.transformer_lm import TransformerLanguageModel

    torch.manual_seed(seed)
    m = TransformerLanguageModel(d, embed_dim=dim, ffn_embed_dim=2 * dim, layers=layers, attention_heads=heads,
                                 max_target_positions=max_pos, share_decoder_input_output_embed=(seed % 2 == 0))
    for p in m.parameters():  # LayerNorm and biases away from their initial 1 / 0, so every parameter matters
        p.data.add_(0.1 * torch.randn_like(p))
    return m.finalize_(device).eval()


def tlm_teacher_forced(lm, dtype=torch.float64):
    """Prefixes (LM indexing, each starting with eos) -> log-softmax of the next token [n, V_lm], through
    oracle/decoder.py:decoder_forward (enc None) on the LM's bf16-rounded parameters."""
    from oracle.decoder import decoder_forward

    sd = {k: v.detach().cpu().float().bfloat16().to(dtype) for k, v in lm.state_dict().items() if k.startswith("decoder.")}
    c = lm.cfg
    cfg = dict(pad=c["pad"], dec_embed_dim=c["embed_dim"], dec_heads=c["heads"], dec_layers=c["layers"], dropout=0.0,
               attention_dropout=0.0, activation_dropout=0.0, share_decoder_input_output_embed=c["share_input_output_embed"])

    def fn(prefixes):
        U = max(len(p) for p in prefixes)
        tok = torch.full((len(prefixes), U), c["pad"], dtype=torch.long)
        for i, p in enumerate(prefixes):
            tok[i, :len(p)] = torch.tensor(p)
        with torch.no_grad():
            out = decoder_forward(sd, cfg, tok, None, None)
        last = torch.tensor([len(p) - 1 for p in prefixes])
        return torch.log_softmax(out[torch.arange(len(prefixes)), last].double(), -1)

    return fn


def lm_oracle_fn(lm, V, eos, lm_blank):
    """oracle/ctc_beam.py's lm_fn: prefix (CTC ids) -> float64 log P_LM(. | eos + prefix) over the CTC vocabulary."""
    tf = tlm_teacher_forced(lm)
    col = lambda v: v - 1 if (lm_blank >= 0 and v > lm_blank) else v  # noqa: E731
    cache = {}

    def fn(y):
        if y not in cache:
            lp = tf([[col(eos)] + [col(v) for v in y]])[0].numpy()
            if lm_blank >= 0:
                lp = np.insert(lp, lm_blank, -np.inf)
            cache[y] = lp[:V]
        return cache[y]

    return fn


def random_frames(N, T, V_lm, seed, mode="random", beam=None):
    """T frames of (new_order, grown, fed) int32 [N] as the search emits them: new_order within each sentence's beam."""
    rs = np.random.RandomState(seed)
    beam = beam or N
    out = []
    for t in range(T):
        base = np.arange(N) // beam * beam
        no = base + rs.randint(0, beam, N)
        gr = (rs.rand(N) < 0.5).astype(np.int32)
        if mode == "all_grow":
            gr[:] = 1
        elif mode == "none_grow":
            gr[:] = 0
        elif mode == "one_parent":
            no = base + (t % beam)
        fed = rs.randint(3, V_lm, N)
        out.append(tuple(torch.tensor(a, dtype=torch.int32) for a in (no, gr, fed)))
    return out


def simulate_paths(frames, N, eos):
    """Host statement of the path tables: per row (cells, tokens) after each frame; slot 0 = every row's eos."""
    paths = [([n], [eos]) for n in range(N)]
    hist = [paths]
    for f, (no, gr, fed) in enumerate(frames):
        slot = f + 1
        new = []
        for n in range(N):
            c, tk = paths[int(no[n])]
            new.append((c + [slot * N + n], tk + [int(fed[n])]) if gr[n] else (c, tk))
        paths = new
        hist.append(paths)
    return hist


@pytest.fixture
def cpu_ops(monkeypatch):
    from espresso_b200 import ops
    from oracle import ctc_beam_ops, ops_ref, prefix_decode_ops

    for mod in (ops_ref, ctc_beam_ops, prefix_decode_ops):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                monkeypatch.setattr(ops, name, getattr(mod, name))


# ---- constructor ---------------------------------------------------------------------------------------------------
def test_vocabulary_with_and_without_the_blank_is_accepted():
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict()
    dec = CTCDecoder(d, blank_idx=0, beam_size=4, lm_model=tlm(d))
    assert dec.transformer and dec.lm_blank == -1
    dec = CTCDecoder(d, blank_idx=0, beam_size=4, lm_model=tlm(_dict(bos=False)))  # one symbol short: no blank
    assert dec.transformer and dec.lm_blank == 0
    with pytest.raises(ValueError, match="LM vocabulary"):
        CTCDecoder(d, blank_idx=0, beam_size=4, lm_model=tlm(_dict(n_sym=7)))


def test_transformer_lm_refusals():
    """What stays refused next to the Transformer LM (tests/test_ctc_beam_search.py covers the KenLM path, a lexicon
    without an n-gram LM and the LSTM word LM)."""
    from espresso_b200.models import TensorizedLookaheadLanguageModel
    from espresso_b200.models.transformer_lm import TransformerLanguageModel
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict()
    raw = TransformerLanguageModel(d, embed_dim=16, ffn_embed_dim=32, layers=1, attention_heads=2)
    with pytest.raises(NotImplementedError, match="finalize_"):  # no native engine yet
        CTCDecoder(d, beam_size=4, lm_model=raw)
    assert CTCDecoder(d, beam_size=4, lm_model=raw.finalize_(torch.device("cpu"))).transformer
    with pytest.raises(NotImplementedError, match="lexicon"):  # a lexicon constrains an n-gram search only
        CTCDecoder(d, beam_size=4, lm_model=tlm(d), lexicon="lexicon.txt")
    wt = tlm(d)
    wt.is_wordlm = True
    with pytest.raises(NotImplementedError, match="word"):
        CTCDecoder(d, beam_size=4, lm_model=wt)
    la = TensorizedLookaheadLanguageModel.__new__(TensorizedLookaheadLanguageModel)
    with pytest.raises(NotImplementedError, match="TensorizedLookaheadLanguageModel"):
        CTCDecoder(d, beam_size=4, lm_model=la)


def test_too_few_lm_positions_are_refused(cpu_ops):
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict()
    V = len(d)
    dec = CTCDecoder(d, blank_idx=0, beam_size=2, lm_model=tlm(d, max_pos=12), lm_weight=0.5)
    x = _logits(1, 11, V, seed=0)
    with pytest.raises(ValueError, match="11 encoder frames need 13 LM positions.*max_target_positions = 12"):
        dec.search(x, V, torch.tensor([11]))
    dec.search(x[:, :10], V, torch.tensor([10]))  # T' + 2 = 12 fits


def test_build_generator_routes_a_ctc_model_with_a_transformer_lm():
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict()
    task = _task(d)
    model = _FakeCTC(_logits(1, 3, len(d), seed=1), torch.tensor([3]), len(d))
    lm = tlm(d)
    g = task.build_generator([model], Namespace(beam=4, lm_weight=0.4, word_score=0.3),
                             extra_gen_cls_kwargs={"lm_model": lm, "lm_weight": 0.4, "eos_factor": 1.5})
    assert isinstance(g, CTCDecoder) and g.transformer and g.lm_model is lm and g.lm_weight == 0.4 and g.word_score == 0.3


# ---- the path tables and the prefix step over oracle/ops_ref ---------------------------------------------------------
def test_update_paths_statement_matches_the_host_simulation():
    from oracle.prefix_decode_ops import decode_update_paths

    N, T = 6, 9
    frames = random_frames(N, T, 10, seed=3, beam=3)
    hist = simulate_paths(frames, N, eos=2)
    cells = torch.full((T + 1, N), -7, dtype=torch.int32)
    ln = torch.zeros(N, dtype=torch.int32)
    c2, l2, pos = cells.clone(), ln.clone(), torch.empty(N, dtype=torch.int32)
    decode_update_paths(cells, ln, c2, l2, torch.arange(N, dtype=torch.int32), torch.ones(N, dtype=torch.int32), 0, pos)
    cells, ln, c2, l2 = c2, l2, cells, ln
    assert pos.tolist() == [0] * N
    for f, (no, gr, _) in enumerate(frames):
        decode_update_paths(cells, ln, c2, l2, no, gr, f + 1, pos)
        assert pos.tolist() == [int(ln[int(p)]) for p in no]
        cells, ln, c2, l2 = c2, l2, cells, ln
        for n, (c, _) in enumerate(hist[f + 1]):
            assert int(ln[n]) == len(c) and cells[: len(c), n].tolist() == c


@pytest.mark.parametrize("lm_blank", [False, True])
def test_prefix_step_over_ops_ref_matches_teacher_forcing(cpu_ops, lm_blank):
    d = _dict(n_sym=11, bos=not lm_blank)
    lm = tlm(d, seed=int(lm_blank) + 1)
    V_lm = len(d)
    bsz, beam, T = 2, 3, 7
    N = bsz * beam
    tf = tlm_teacher_forced(lm)
    frames = random_frames(N, T, V_lm, seed=5 + int(lm_blank), beam=beam)
    hist = simulate_paths(frames, N, d.eos())
    st = lm.init_prefix_state(bsz, beam, T)
    ix = torch.arange(N, dtype=torch.int32)
    rows = lm.prefix_step(0, torch.full((N,), d.eos(), dtype=torch.int32), torch.ones_like(ix), ix, st)
    err, scale = 0.0, 0.0
    for f in range(T + 1):
        if f > 0:
            no, gr, fed = frames[f - 1]
            new_rows = lm.prefix_step(f, fed, gr, no, st)
            rows = torch.where(gr.view(N, 1) != 0, new_rows, rows.index_select(0, no.long()))
        ref = tf([tk for _, tk in hist[f]])
        got = torch.log_softmax(rows[:, :V_lm].double(), -1)
        err = max(err, float((got - ref).abs().max()))
        scale = max(scale, float(rows[:, :V_lm].float().abs().max()))
    assert err <= LOGIT_ULPS * max(1.0, scale), (err, scale)


def test_host_search_over_ops_ref_matches_the_oracle(cpu_ops):
    """The decoder's frame loop over the statements, against oracle/ctc_beam.search with the teacher-forced LM: the LM
    is bf16 in the loop and float64 in the oracle, so hypotheses must match where the oracle's margins exceed that."""
    from oracle import ctc_beam as O

    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict()
    V = len(d)
    lm = tlm(_dict(bos=False), seed=2)
    beam, K, thr, lw, ws = 4, 5, 6.0, 0.47, 0.3
    dec = CTCDecoder(d, blank_idx=0, beam_size=beam, lm_model=lm, lm_weight=lw, word_score=ws, beam_size_token=K,
                     beam_threshold=thr, nbest=3, print_alignment=True)
    B, T = 3, 9
    x = _logits(B, T, V, seed=7, peaked=True)
    lens = torch.tensor([9, 4, 0])
    tokens, lens_o, scores, frames = dec.search(x, V, lens)
    lm_fn = lm_oracle_fn(lm, V, d.eos(), 0)
    n_exact = 0
    for b in range(B):
        ref = O.search(x[b, : int(lens[b]), :V].double().numpy(), beam, K, 0, (d.pad(), d.eos(), d.unk()), thr, lm_fn, lw, ws,
                       d.eos())
        sc = [r[1] for r in ref]
        for r in range(min(3, len(ref))):
            gap = min(sc[r - 1] - sc[r] if r > 0 else math.inf, sc[r] - sc[r + 1] if r + 1 < len(sc) else math.inf)
            n = int(lens_o[b, r])
            if gap > 0.05:
                assert tuple(tokens[b, r, :n].tolist()) == ref[r][0] and tuple(frames[b, r, :n].tolist()) == ref[r][2]
                assert abs(float(scores[b, r]) - sc[r]) <= 0.02 * max(1.0, abs(sc[r]))
                n_exact += 1
    assert n_exact >= 3
    assert int(lens_o[2, 0]) == 0 and scores[2, 0] > -math.inf  # in_len 0: the empty prefix, scored with P_LM(eos | eos)


def test_recognize_ctc_with_transformer_lm(tmp_path, cpu_ops, monkeypatch):
    """recognize() on a CTC task with lms=[transformer_lm]: H- lines carry the decoder's scores and the LM (at a high
    weight) changes the hypotheses."""
    import os

    from test_input_pipeline import _corpus

    from espresso_b200.data.asr_dictionary import AsrDictionary
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel
    from espresso_b200.speech_recognize import recognize
    from espresso_b200.tasks.speech_recognition import SpeechRecognitionEspressoConfig, SpeechRecognitionEspressoTask
    from espresso_b200.tools.ctc_decoder import CTCDecoder

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
        encoder=dict(embed_dim=32, ffn_embed_dim=64, layers=1, attention_heads=2, normalize_before=True, learned_pos=False,
                     relative_positional_embeddings=True, layer_type="transformer")))
    m = SpeechTransformerEncoderModel.build_model(mcfg, task).finalize_(torch.device("cpu"))
    m.frontend = OnTheFlyFbank(None, None)
    seen = []
    orig = CTCDecoder.generate

    def spy(self, models, sample, **kw):
        assert self.transformer
        out = orig(self, models, sample, **kw)
        seen.extend(h[0]["score"] for h in out)
        return out

    lm = tlm(d, seed=1)
    run = lambda lms, w: recognize(task, [m], subset="test", gen_args=Namespace(beam=4, lm_weight=w), lms=lms,  # noqa: E731
                                   max_tokens=None, max_sentences=2, device="cpu")
    plain = run(None, 0.0)
    monkeypatch.setattr(CTCDecoder, "generate", spy)
    fused = run([lm], 4.0)
    h_lines = [l for l in fused["lines"] if l.startswith("H-")]
    assert len(h_lines) == len(man) == len(seen)
    for l, s in zip(h_lines, seen):
        assert float(l.split("\t")[2]) == s / math.log(2) and s < 0.0
    hyp = lambda out: {l.split("\t")[0]: l.split("\t")[1] for l in out["lines"] if l.startswith("H-")}  # noqa: E731
    assert hyp(plain) != hyp(fused)
