"""CPU: the CTC prefix beam search.  oracle/ctc_beam.py is pinned against exact CTC marginals (F.ctc_loss in float64 and
an exhaustive enumeration of alignments) and a table LM; the host orchestration of espresso_b200.tools.ctc_decoder runs over
oracle/ops_ref + oracle/ctc_beam_ops (the plain statement of the three kernels) and must reproduce the oracle;
build_generator routing, the refusals and the recognize() loop on a CTC task with an LSTM LM."""
import copy
import itertools
import math
from argparse import Namespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ctc_beam as O


def _ctc_logp(x, y, blank):
    """log P_ctc(y | x) in float64 through F.ctc_loss (reduction none)."""
    lp = torch.log_softmax(torch.as_tensor(x, dtype=torch.float64), -1)[:, None]
    tg = torch.tensor([list(y)], dtype=torch.long) if y else torch.zeros(1, 0, dtype=torch.long)
    return -F.ctc_loss(lp, tg, torch.tensor([lp.shape[0]]), torch.tensor([len(y)]), blank=blank, reduction="none",
                       zero_infinity=False).item()


def _enumerate(x, blank):
    """Every collapsed label sequence with its log-probability, summed over all alignments (float64)."""
    lp = O.log_softmax(x)
    T, V = lp.shape
    acc = {}
    for path in itertools.product(range(V), repeat=T):
        y, prev = [], None
        for p in path:
            if p != prev and p != blank:
                y.append(p)
            prev = p
        s = sum(lp[t, p] for t, p in enumerate(path))
        acc[tuple(y)] = np.logaddexp(acc.get(tuple(y), -np.inf), s)
    return acc


@pytest.mark.parametrize("T,V,blank,seed", [(4, 3, 0, 0), (5, 3, 2, 1), (6, 3, 1, 2), (4, 4, 0, 3), (3, 5, 3, 4)])
def test_oracle_without_pruning_is_exact_ctc(T, V, blank, seed):
    rs = np.random.RandomState(seed)
    x = rs.randn(T, V) * 1.5
    hyps = O.search(x, beam=10 ** 6, K=V, blank=blank)
    exact = _enumerate(x, blank)
    assert len(hyps) == len(exact)  # every reachable prefix survives
    for y, s, fr in hyps:
        assert abs(s - _ctc_logp(x, y, blank)) < 1e-10
        assert abs(s - exact[y]) < 1e-10
        assert len(fr) == len(y) and list(fr) == sorted(fr)
    ranked = sorted(exact.items(), key=lambda kv: -kv[1])
    assert [h[0] for h in hyps] == [k for k, _ in ranked]
    # repeated tokens need a blank in between: they are reachable only when T allows it
    rep = [y for y, _, _ in hyps if any(a == b for a, b in zip(y, y[1:]))]
    assert rep and all(len(y) + sum(a == b for a, b in zip(y, y[1:])) <= T for y in rep)


@pytest.mark.parametrize("lm_weight,word_score", [(0.47, 0.0), (0.8, -0.3), (1.3, 0.7)])
def test_oracle_with_table_lm_is_exact(lm_weight, word_score):
    rs = np.random.RandomState(5)
    T, V, blank, eos = 4, 5, 0, 4
    x = rs.randn(T, V)
    table = O.log_softmax(rs.randn(V, V))  # bigram LM, context = last token or eos

    def lm_fn(y):
        return table[y[-1] if y else eos]

    hyps = O.search(x, beam=10 ** 6, K=V, blank=blank, exclude=(eos,), lm_fn=lm_fn, lm_weight=lm_weight,
                    word_score=word_score, eos=eos)
    assert sorted(h[0] for h in hyps) == sorted(y for y in _enumerate(x, blank) if eos not in y)
    for y, s, _ in hyps:
        ctx = (eos,) + tuple(y)
        lm = sum(table[a, b] for a, b in zip(ctx, y)) + table[ctx[-1], eos]
        assert abs(s - (_ctc_logp(x, y, blank) + lm_weight * lm + word_score * len(y))) < 1e-10
    assert [h[1] for h in hyps] == sorted((h[1] for h in hyps), reverse=True)


def test_oracle_pruning_keeps_the_best_and_orders_ties_by_index():
    x = np.zeros((3, 4))  # every token equally likely: ties everywhere
    hyps = O.search(x, beam=3, K=2, blank=0)
    assert len(hyps) == 3
    hyps_thr = O.search(np.random.RandomState(0).randn(6, 6) * 4, beam=8, K=5, blank=0, threshold=1.0)
    assert hyps_thr[0][1] - hyps_thr[-1][1] <= 1.0 + 1e-12


# ---- host orchestration over oracle/ops_ref + oracle/ctc_beam_ops ----------------------------------------------------
def _dict(n_sym=9, bos=True):
    from espresso_b200.data.asr_dictionary import AsrDictionary

    d = AsrDictionary(enable_bos=bos)
    for i in range(n_sym):
        d.add_symbol("abcdefghijklmnopqrstuvwxyz"[i] if i < 26 else "s%d" % i)
    return d


def _lstm_lm(d, seed=0, hidden=24):
    from espresso_b200.models.lstm_lm import LSTMLanguageModelEspresso, LSTMLanguageModelEspressoConfig

    torch.manual_seed(seed)
    cfg = LSTMLanguageModelEspressoConfig(dropout=0.0, decoder_embed_dim=16, decoder_hidden_size=hidden, decoder_layers=2,
                                          decoder_out_embed_dim=hidden)
    return LSTMLanguageModelEspresso.build_model(cfg, Namespace(target_dictionary=d)).eval()


def lm_oracle_fn(lm, V, eos, lm_blank):
    """Prefix -> float64 log P_LM(. | eos + prefix) over the CTC vocabulary, from a float64 copy of the LM (teacher forced)."""
    lm64 = copy.deepcopy(lm).double().eval()
    col = lambda v: v - 1 if (lm_blank >= 0 and v > lm_blank) else v  # noqa: E731
    cache = {}

    def fn(y):
        if y not in cache:
            src = torch.tensor([[col(eos)] + [col(v) for v in y]])
            with torch.no_grad():
                lp = torch.log_softmax(lm64(src)[0][0, -1].double(), -1).numpy()
            if lm_blank >= 0:
                lp = np.insert(lp, lm_blank, -np.inf)
            cache[y] = lp[:V]
        return cache[y]

    return fn


@pytest.fixture
def cpu_ops(monkeypatch):
    from espresso_b200 import ops
    from oracle import ctc_beam_ops, ops_ref

    for mod in (ops_ref, ctc_beam_ops):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                monkeypatch.setattr(ops, name, getattr(mod, name))


def _logits(B, T, V, seed, ld=None, peaked=False):
    rs = np.random.RandomState(seed)
    ld = ld or (V + 7) // 8 * 8
    x = rs.randn(B, T, ld) * (3.0 if peaked else 1.0)
    return torch.from_numpy(x).float().bfloat16()


@pytest.mark.parametrize("with_lm", [False, True])
def test_host_search_over_ops_ref_matches_the_oracle(cpu_ops, with_lm):
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict()
    V = len(d)
    lm = _lstm_lm(_dict(bos=False)) if with_lm else None  # LM vocabulary without the blank
    beam, K, thr, lw, ws = 4, 5, 6.0, 0.47, 0.3
    dec = CTCDecoder(d, blank_idx=0, beam_size=beam, lm_model=lm, lm_weight=lw, word_score=ws, beam_size_token=K,
                     beam_threshold=thr, nbest=3, print_alignment=True)
    B, T = 3, 9
    x = _logits(B, T, V, seed=7)
    lens = torch.tensor([9, 4, 0])
    tokens, lens_o, scores, frames = dec.search(x, V, lens)
    lm_fn = lm_oracle_fn(lm, V, d.eos(), 0) if with_lm else None
    for b in range(B):
        ref = O.search(x[b, : int(lens[b]), :V].double().numpy(), beam, K, 0, (d.pad(), d.eos(), d.unk()), thr, lm_fn,
                       lw if with_lm else 0.0, ws, d.eos())
        for r in range(3):
            if r >= len(ref):
                assert scores[b, r] == -math.inf
                continue
            y, s, fr = ref[r]
            n = int(lens_o[b, r])
            assert tuple(tokens[b, r, :n].tolist()) == y and (tokens[b, r, n:] == d.pad()).all()
            assert tuple(frames[b, r, :n].tolist()) == fr
            assert abs(float(scores[b, r]) - s) <= 1e-5 * max(1.0, abs(s))
    assert int(lens_o[2, 0]) == 0 and abs(float(scores[2, 0])) <= (1e-5 if not with_lm else 30)  # in_len 0: empty prefix


class _FakeCTC:
    """Stands in for a CTC model: returns fixed logits in the model's output dict."""

    def __init__(self, logits, lens, V):
        self.logits, self.lens, self.V = logits, lens, V

    def eval(self):
        return self

    def __call__(self, **unused):
        return {"b200_out": self.logits, "encoder_out": [torch.zeros(1, 1, self.V)], "src_lengths": [self.lens]}


def _task(d):
    from espresso_b200.tasks.speech_recognition import SpeechRecognitionEspressoConfig, SpeechRecognitionEspressoTask

    return SpeechRecognitionEspressoTask(SpeechRecognitionEspressoConfig(criterion_name="ctc_loss"), d, feat_dim=80)


def test_build_generator_routing_and_greedy_unchanged(cpu_ops):
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict()
    V = len(d)
    task = _task(d)
    x = _logits(3, 11, V, seed=3, peaked=True)
    lens = torch.tensor([11, 6, 1])
    model = _FakeCTC(x, lens, V)
    g = task.build_generator([model], Namespace(beam=1))
    assert isinstance(g, CTCDecoder) and g.greedy
    tokens, scores, align = g.decode([model], {"net_input": {}})
    # the greedy statement: argmax, collapse repeats, drop blanks
    am = x[..., :V].float().argmax(-1)
    for b in range(3):
        seq = torch.unique_consecutive(am[b, : int(lens[b])])
        seq = seq[seq != 0]
        assert tokens[b, : seq.numel()].tolist() == seq.tolist() and (tokens[b, seq.numel():] == d.pad()).all()
    assert scores is None and align is None
    assert [h[0]["score"] for h in g.generate([model], {"net_input": {}})] == [0.0] * 3
    # the validation decoder stays greedy
    assert task.build_decoder_for_validation(model).greedy
    # beam > 1, or an LM at beam 1, gives the prefix beam search
    g4 = task.build_generator([model], Namespace(beam=4, lm_weight=0.5, word_score=0.2, nbest=2))
    assert not g4.greedy and g4.beam_size == 4 and g4.lm_weight == 0.5 and g4.word_score == 0.2 and g4.nbest == 2
    lm = _lstm_lm(d)
    g1 = task.build_generator([model], Namespace(beam=1), extra_gen_cls_kwargs={"lm_model": lm, "lm_weight": 0.3,
                                                                                 "eos_factor": 1.5})
    assert not g1.greedy and g1.lm_model is lm and g1.lm_blank == -1
    hy = g4.generate([model], {"net_input": {}})
    assert len(hy) == 3 and all(1 <= len(h) <= 2 for h in hy)
    assert all(h[0]["score"] >= h[-1]["score"] for h in hy)
    tb, sb, _ = g4.decode([model], {"net_input": {}})
    assert torch.equal(sb, torch.tensor([h[0]["score"] for h in hy]))
    assert all(d.unk() not in h["tokens"].tolist() for hs in hy for h in hs)  # unk is excluded by default, as in the reference


def test_unsupported_lms_and_lexicon_are_refused():
    from espresso_b200.models.transformer_lm import TransformerLanguageModel
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = _dict()
    with pytest.raises(NotImplementedError, match="KenLM"):
        CTCDecoder(d, beam_size=4, lm_model="/path/to/lm.arpa")
    with pytest.raises(NotImplementedError, match="lexicon"):
        CTCDecoder(d, beam_size=4, lexicon="lexicon.txt")
    tlm = TransformerLanguageModel(d, embed_dim=16, ffn_embed_dim=32, layers=1, attention_heads=2)
    with pytest.raises(NotImplementedError, match="TransformerLanguageModel"):
        CTCDecoder(d, beam_size=4, lm_model=tlm)
    wlm = _lstm_lm(d)
    wlm.is_wordlm = True
    with pytest.raises(NotImplementedError, match="LSTM subword LM"):
        CTCDecoder(d, beam_size=4, lm_model=wlm)


def test_recognize_ctc_with_lstm_lm(tmp_path, cpu_ops, monkeypatch):
    """recognize() on a CTC task: manifest -> batches -> Conformer-free encoder -> prefix beam search with the LSTM LM ->
    H- lines whose scores are the decoder's natural-log scores / ln 2; the LM changes the hypotheses."""
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
        out = orig(self, models, sample, **kw)
        seen.extend(h[0]["score"] for h in out)
        return out

    monkeypatch.setattr(CTCDecoder, "generate", spy)
    lm = _lstm_lm(d, seed=1)
    run = lambda lms, w: recognize(task, [m], subset="test", gen_args=Namespace(beam=4, lm_weight=w), lms=lms,  # noqa: E731
                                   max_tokens=None, max_sentences=2, device="cpu")
    plain = run(None, 0.0)
    seen.clear()
    fused = run([lm], 4.0)
    h_lines = [l for l in fused["lines"] if l.startswith("H-")]
    assert len(h_lines) == len(man) == len(seen)
    for l, s in zip(h_lines, seen):
        assert float(l.split("\t")[2]) == s / math.log(2) and s < 0.0
    hyp = lambda out: {l.split("\t")[0]: l.split("\t")[1] for l in out["lines"] if l.startswith("H-")}  # noqa: E731
    assert hyp(plain) != hyp(fused)
