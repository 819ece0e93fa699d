"""CPU: the encoder attention of the beam search (`print_alignment`).

The host SequenceGenerator, with oracle/ops_ref.py + oracle/beam_attention.py standing in for the native ops and the fp32
model oracle.beam_attention.Fp32EncDec, reproduces the REAL reference generator's hypotheses and attention matrices recorded
in tests/golden/beam_attention.npz (beam 4 with the full n-best, a two-model ensemble, eos forced at max_len); with the flag
off nothing changes; the product Transformer records the same matrices through its incremental decoder; recognize() plots
the best hypothesis of every utterance of an attention model and nothing for CTC."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from oracle import beam_attention as OA  # noqa: E402
from oracle import ops_ref  # noqa: E402

CASES = {"beam4": 1, "ensemble": 2, "maxlen": 1}
ATT_BOUND = 0.04  # |bf16 attention - fp32|, abs, of the product model (0.031 reached; its queries are scaled up to 80x)
GEN_KW = {"beam4": dict(beam_size=4, max_len_a=0.0, max_len_b=40), "ensemble": dict(beam_size=4, max_len_a=0.0, max_len_b=40),
          "maxlen": dict(beam_size=4, max_len_a=0.0, max_len_b=3)}


@pytest.fixture
def cpu_ops(monkeypatch):
    from espresso_b200 import ops

    for mod in (ops_ref, OA):
        for name in dir(mod):
            if not name.startswith("_") and callable(getattr(mod, name)) and hasattr(ops, name):
                monkeypatch.setattr(ops, name, getattr(mod, name))


class _Dict:
    def __len__(self):
        return 50

    def pad(self):
        return 1

    def eos(self):
        return 2

    def unk(self):
        return 3


def _fixture(golden_dir):
    g = np.load(os.path.join(golden_dir, "beam_attention.npz"))
    e = np.load(os.path.join(golden_dir, "encdec_transformer.npz"))
    sd1 = OA.search_model({k[3:]: e[k] for k in e.files if k.startswith("sd.")})
    sd2 = OA.perturbed(sd1)
    for sd, key in ((sd1, "sd1_abs_sum"), (sd2, "sd2_abs_sum")):
        assert abs(sum(np.abs(v).astype(np.float64).sum() for v in sd.values()) / float(g[key]) - 1) < 1e-6
    return g, [sd1, sd2]


class _Npz:
    """The encdec fixture with its weights replaced (what _build_encdec reads)."""

    def __init__(self, sd, base):
        self.d = {"sd." + k: v for k, v in sd.items()}
        self.base = base
        self.files = list(self.d)

    def __getitem__(self, k):
        return self.d[k] if k in self.d else self.base[k]


def _sample(g):
    return {"net_input": {"src_tokens": torch.from_numpy(g["feats"]), "src_lengths": torch.from_numpy(g["lens"])}}


@pytest.mark.parametrize("case", sorted(CASES))
def test_host_generator_reproduces_reference_attention(case, golden_dir, cpu_ops):
    from espresso_b200.sequence_generator import SequenceGenerator

    g, sds = _fixture(golden_dir)
    models = [OA.Fp32EncDec(sd) for sd in sds[: CASES[case]]]
    got = SequenceGenerator(models, _Dict(), print_alignment="hard", **GEN_KW[case]).generate(models, _sample(g))
    Tp = g["%s_b0_k0_attention" % case].shape[0]
    worst = 0.0
    for b, hyps in enumerate(got):
        assert len(hyps) == int(g["%s_b%d_n" % (case, b)])
        for k, h in enumerate(hyps):
            key = "%s_b%d_k%d_" % (case, b, k)
            assert h["tokens"].tolist() == g[key + "tokens"].tolist(), key
            assert abs(float(h["score"]) - float(g[key + "score"])) < 1e-5
            assert h["alignment"] is None and h["attention"].dtype == torch.float32
            assert h["attention"].shape == (Tp, len(h["tokens"]))
            worst = max(worst, float((h["attention"] - torch.from_numpy(g[key + "attention"])).abs().max()))
    assert worst < 1e-5, worst


def test_flag_off_changes_nothing(golden_dir, cpu_ops):
    from espresso_b200.sequence_generator import SequenceGenerator

    g, sds = _fixture(golden_dir)
    m = OA.Fp32EncDec(sds[0])
    on = SequenceGenerator([m], _Dict(), print_alignment=True, **GEN_KW["maxlen"]).generate([m], _sample(g))
    off = SequenceGenerator([m], _Dict(), **GEN_KW["maxlen"]).generate([m], _sample(g))
    for a, b in zip(on, off):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            assert y["attention"] is None and x["attention"] is not None
            assert torch.equal(x["tokens"], y["tokens"]) and torch.equal(x["score"], y["score"])
            assert torch.equal(x["positional_scores"], y["positional_scores"])


def test_product_transformer_records_attention_through_incremental_decoder(golden_dir, cpu_ops):
    """The product model (bf16 statement of the kernels on the CPU): alignments on vs off give identical hypotheses; every
    column is a distribution over the utterance's frames (padded frames exactly 0); the matrices follow the fp32 oracle
    teacher-forced along the same tokens to bf16 accuracy."""
    from test_host_orchestration import _build_encdec

    from espresso_b200.sequence_generator import SequenceGenerator

    g, sds = _fixture(golden_dir)
    m = _build_encdec(_Npz(sds[0], np.load(os.path.join(golden_dir, "encdec_transformer.npz")))).finalize_(torch.device("cpu"))
    m.eval()
    kw = dict(beam_size=3, max_len_a=0.0, max_len_b=5)
    on = SequenceGenerator([m], _Dict(), print_alignment=True, **kw).generate([m], _sample(g))
    off = SequenceGenerator([m], _Dict(), **kw).generate([m], _sample(g))
    ref = OA.Fp32EncDec(sds[0])
    enc = ref.forward_encoder(_sample(g)["net_input"])
    Tp = enc["enc"].shape[1]
    out_lens = m.encoder.output_lengths(torch.from_numpy(g["lens"])).tolist()
    worst, sep = 0.0, float("inf")
    for b, (a, c) in enumerate(zip(on, off)):
        assert len(a) == len(c)
        for x, y in zip(a, c):
            assert torch.equal(x["tokens"], y["tokens"]) and torch.equal(x["score"], y["score"]) and y["attention"] is None
            att = x["attention"]
            assert att.shape == (Tp, len(x["tokens"]))
            assert torch.all(att[out_lens[b]:] == 0)
            assert (att.sum(0) - 1).abs().max() < 1e-5
            prefix = torch.cat([torch.tensor([2]), x["tokens"]])
            off_uniform = 0.0
            for t in range(len(x["tokens"])):
                _, r = OA.decoder_step(ref.sd, prefix[None, : t + 1], enc["enc"][b:b + 1],
                                       None if enc["pad"] is None else enc["pad"][b:b + 1])
                worst = max(worst, (att[:, t] - r[0]).abs().max().item())
                uniform = (torch.arange(Tp) < out_lens[b]).float() / out_lens[b]
                off_uniform = max(off_uniform, (uniform - r[0]).abs().max().item())
            sep = min(sep, off_uniform)  # how far a matrix of uniform rows would be off
    print("product transformer on the CPU: worst |att - fp32| %.3g, uniform rows off by >= %.3g" % (worst, sep))
    assert worst < ATT_BOUND, worst
    assert sep > ATT_BOUND, sep  # a matrix of uniform rows fails


def _attention_task(tmp_path, criterion):
    from test_input_pipeline import _corpus

    from espresso_b200.tasks.speech_recognition import SpeechRecognitionEspressoConfig, SpeechRecognitionEspressoTask

    d, man = _corpus(tmp_path, n=5, fmt="wave")
    os.rename(str(tmp_path / "train.json"), str(tmp_path / "test.json"))
    if criterion == "ctc_loss":  # the CTC decoder strips <s>: a dictionary that has one
        from espresso_b200.data.asr_dictionary import AsrDictionary

        d0, d = d, AsrDictionary(enable_bos=True)
        for sym in d0.symbols[d0.nspecial:]:
            d.add_symbol(sym)
        d.space_index = d.index("<space>")
        d.build_bpe("characters_asr")
    cfg = SpeechRecognitionEspressoConfig(criterion_name=criterion, data=str(tmp_path), autoregressive=criterion != "ctc_loss")
    return SpeechRecognitionEspressoTask(cfg, d, feat_dim=80), man


def test_recognize_plots_the_best_hypothesis_attention(tmp_path, cpu_ops, monkeypatch):
    from argparse import Namespace

    from espresso_b200 import speech_recognize
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerModelBase
    from espresso_b200.sequence_generator import SequenceGenerator

    task, man = _attention_task(tmp_path, "label_smoothed_cross_entropy_v2")
    torch.manual_seed(3)
    mcfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, layernorm_embedding=False, max_target_positions=64,
        encoder=dict(embed_dim=64, ffn_embed_dim=128, layers=1, attention_heads=4, normalize_before=True, learned_pos=False,
                     relative_positional_embeddings=True, layer_type="transformer"),
        decoder=dict(embed_dim=64, ffn_embed_dim=128, layers=1, attention_heads=4, normalize_before=True, learned_pos=False,
                     relative_positional_embeddings=False, input_dim=64, output_dim=64)))
    m = SpeechTransformerModelBase.build_model(mcfg, task).finalize_(torch.device("cpu"))
    m.frontend = OnTheFlyFbank(None, None)
    calls, best = [], {}
    monkeypatch.setattr(speech_recognize, "plot_attention", lambda a, s, u, d: calls.append((a.clone(), s, u, d)))
    orig = SequenceGenerator.generate

    def spy(self, models, sample, **kw):
        out = orig(self, models, sample, **kw)
        waves, n = sample["net_input"]["src_tokens"], sample["net_input"]["src_lengths"]
        frames = m.encoder.output_lengths(1 + torch.div(n - 400, 160, rounding_mode="floor"))
        assert waves.dim() == 2
        for i, hyps in enumerate(out):
            best[sample["utt_id"][i]] = (hyps[0], int(frames[i]))
        return out

    monkeypatch.setattr(SequenceGenerator, "generate", spy)
    args = Namespace(beam=2, max_len_a=0.0, max_len_b=6, lm_weight=0.0)
    res = speech_recognize.recognize(task, [m], subset="test", gen_args=args, max_tokens=None, max_sentences=3, device="cpu",
                                     print_alignment=True, results_path=str(tmp_path / "res"))
    assert len(calls) == len(man) == len(best)
    h_lines = {l.split("\t")[0][2:]: l.split("\t")[1] for l in res["lines"] if l.startswith("H-")}
    for a, title, utt, save_dir in calls:
        h, L = best[utt]
        assert save_dir == os.path.join(str(tmp_path / "res"), "attn_plots") and os.path.isdir(save_dir)
        assert title == h_lines[utt]
        assert a.shape == (L, len(h["tokens"])) and L < h["attention"].shape[0] + 1
        assert torch.equal(a, h["attention"][:L])
        assert torch.all(h["attention"][L:] == 0) and (a.sum(0) - 1).abs().max() < 1e-5
    with pytest.raises(ValueError, match="results_path"):
        speech_recognize.recognize(task, [m], subset="test", gen_args=args, max_tokens=None, max_sentences=3, device="cpu",
                                   print_alignment=True)


def test_recognize_ctc_makes_no_attention_plot(tmp_path, cpu_ops, monkeypatch):
    from argparse import Namespace

    from espresso_b200 import speech_recognize
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel

    task, man = _attention_task(tmp_path, "ctc_loss")
    torch.manual_seed(4)
    mcfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, layernorm_embedding=False,
        encoder=dict(embed_dim=32, ffn_embed_dim=64, layers=1, attention_heads=2, normalize_before=True, learned_pos=False,
                     relative_positional_embeddings=True, layer_type="transformer")))
    m = SpeechTransformerEncoderModel.build_model(mcfg, task).finalize_(torch.device("cpu"))
    m.frontend = OnTheFlyFbank(None, None)
    monkeypatch.setattr(speech_recognize, "plot_attention", lambda *a: pytest.fail("CTC models have no attention plot"))
    res = speech_recognize.recognize(task, [m], subset="test", gen_args=Namespace(beam=1), max_tokens=None, max_sentences=2,
                                     device="cpu", print_alignment=True)
    assert len([l for l in res["lines"] if l.startswith("H-")]) == len(man)


def test_plot_attention_without_matplotlib_raises_reference_message(tmp_path):
    try:
        import matplotlib  # noqa: F401
        pytest.skip("matplotlib is installed")
    except ImportError:
        pass
    from espresso_b200.tools.utils import plot_attention

    with pytest.raises(ImportError, match="(?s)This function requires matplotlib.*unset --print-alignment"):
        plot_attention(torch.rand(4, 3), "a b", "utt1", str(tmp_path))


def test_speech_lstm_state_yields_no_attention(cpu_ops):
    """A model whose state records no attention (no decode_attention, like speech_lstm) gives attention None."""
    from test_beam_search import _RandomModel

    from espresso_b200.sequence_generator import SequenceGenerator

    class D(_Dict):
        def __len__(self):
            return 9

    m = _RandomModel(9, 1)
    out = SequenceGenerator([m], D(), beam_size=2, max_len_a=0.0, max_len_b=5, print_alignment=True).generate(
        [m], {"net_input": {"src_tokens": torch.zeros(2, 7, dtype=torch.long), "src_lengths": torch.full((2,), 7)}})
    assert all(h["attention"] is None for hs in out for h in hs)
    assert math.isfinite(float(out[0][0]["score"]))
