"""CPU: the speech models' input side, with the oracle's per-op reference (oracle/ops_ref.py) patched in for the CUDA ops.
One fbank frame count, stated in ops.py only; raw waveforms reach the encoder the same way through every entry point:
`forward`, `forward_encoder` and the transducer decoders."""
import ast
import os

import numpy as np
import pytest
import torch

from oracle import ops_ref

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "espresso_b200")


@pytest.fixture()
def cpu_ops(monkeypatch):
    from espresso_b200 import ops

    for name in dir(ops_ref):
        if name.startswith("_") or not callable(getattr(ops_ref, name)) or not hasattr(ops, name):
            continue
        monkeypatch.setattr(ops, name, getattr(ops_ref, name))
    return ops


class _Dict:
    def __len__(self):
        return 20

    def pad(self):
        return 1

    def eos(self):
        return 2

    def bos(self):
        return 0

    def index(self, sym):
        return 0


class _Task:
    feat_dim, feat_in_channels, target_dictionary = 80, 1, _Dict()


def _cfg():
    from espresso_b200.models import SpeechTransformerConfig

    return SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, layernorm_embedding=True, max_target_positions=32,
        encoder=dict(embed_dim=32, ffn_embed_dim=64, layers=1, attention_heads=2, normalize_before=True,
                     relative_positional_embeddings=True, layer_type="transformer", conv_channels="[64, 64]",
                     conv_kernel_sizes="[(3, 3), (3, 3)]", conv_strides="[(2, 2), (2, 2)]"),
        decoder=dict(embed_dim=32, ffn_embed_dim=64, layers=1, attention_heads=2, normalize_before=True, input_dim=32,
                     output_dim=32)))


def _models():
    from espresso_b200.models import SpeechTransformerEncoderModel, SpeechTransformerModelBase, SpeechTransformerTransducerModelBase

    torch.manual_seed(0)
    return {
        "encoder": SpeechTransformerEncoderModel.build_model(_cfg(), _Task()),
        "encdec": SpeechTransformerModelBase.build_model(_cfg(), _Task()),
        "transducer": SpeechTransformerTransducerModelBase.build_model(
            _cfg(), _Task(), decoder_hidden_size=32, decoder_layers=1, decoder_embed_dim=32, joint_dim=32),
    }


def _waves():
    n = torch.tensor([6400, 4000, 2900])
    rs = np.random.RandomState(0)
    w = torch.from_numpy(np.round(rs.randn(3, int(n.max())) * 2000).astype(np.float32))
    for i in range(3):
        w[i, int(n[i]):] = 0
    return w, n


def test_num_frames_matches_the_oracle():
    from espresso_b200 import ops
    from oracle import frontend as ofe

    ns = [0, 399, 400, 559, 560, 160000]
    assert [ops.num_frames(n) for n in ns] == [ofe.num_frames(n) for n in ns]
    t = ops.num_frames(torch.tensor(ns, dtype=torch.int64))
    assert t.dtype == torch.int64 and t.tolist() == [ofe.num_frames(n) for n in ns]


def test_frame_count_is_stated_in_ops_only():
    """No line under espresso_b200/ outside ops.py names both the 400-sample window and the 160-sample hop.  The one
    exception is Trainer._bucket_shapes: it pads a waveform's sample count to a bucket of frames, a different rule (one
    frame below 400 samples) that only picks CUDA-graph shapes."""
    found = []
    for d, _, files in os.walk(PKG):
        for f in files:
            path = os.path.join(d, f)
            if not f.endswith(".py") or path == os.path.join(PKG, "ops.py"):
                continue
            src = open(path).read()
            skip = set()
            if f == "trainer.py":
                fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == "_bucket_shapes")
                skip = set(range(fn.lineno, fn.end_lineno + 1))
            for i, line in enumerate(src.splitlines(), 1):
                code = line.split("#")[0]
                if i not in skip and "400" in code and "160" in code:
                    found.append("%s:%d: %s" % (os.path.relpath(path, PKG), i, line.strip()))
    assert not found, "frame counts outside ops.num_frames:\n" + "\n".join(found)


def test_waveform_host_lengths_do_not_change_the_encoding(cpu_ops):
    """Host sample counts (`src_lengths_cpu`) are converted to frames like the device lengths, so giving them changes
    neither the padding mask nor any output: encoder-decoder `forward_encoder` and both transducer decoders."""
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.tools.transducer_beam_search_decoder import TransducerBeamSearchDecoder
    from espresso_b200.tools.transducer_greedy_decoder import TransducerGreedyDecoder

    ms = _models()
    w, n = _waves()
    with_cpu = {"src_tokens": w, "src_lengths": n, "src_lengths_cpu": n.clone()}
    without = {"src_tokens": w, "src_lengths": n}
    for name in ("encdec", "transducer"):
        m = ms[name].finalize_(torch.device("cpu")).eval()
        m.frontend = OnTheFlyFbank(None, None)
        seen = []
        enc_forward = m.encoder.forward
        m.encoder.forward = lambda *a, **kw: seen.append(enc_forward(*a, **kw)) or seen[-1]
        if name == "encdec":
            with torch.no_grad():
                m.forward_encoder(with_cpu)
                m.forward_encoder(without)
        else:
            for dec in (TransducerGreedyDecoder([m], _Dict(), blank=0),
                        TransducerBeamSearchDecoder([m], _Dict(), blank=0, beam_size=2)):
                tok_a, sc_a, _ = dec.decode([m], {"net_input": with_cpu})
                tok_b, sc_b, _ = dec.decode([m], {"net_input": without})
                assert torch.equal(tok_a, tok_b) and torch.equal(sc_a, sc_b), type(dec).__name__
        assert len(seen) in (2, 4)
        for a, b in zip(seen[0::2], seen[1::2]):
            assert len(a["encoder_padding_mask"]) == len(b["encoder_padding_mask"]) == 1, name
            assert torch.equal(a["encoder_padding_mask"][0], b["encoder_padding_mask"][0]), name
            assert torch.equal(a["b200_out"], b["b200_out"]), name


def test_waveform_without_front_end_is_refused_everywhere():
    from espresso_b200.tools.transducer_beam_search_decoder import TransducerBeamSearchDecoder
    from espresso_b200.tools.transducer_greedy_decoder import TransducerGreedyDecoder

    ms = {k: m.finalize_(torch.device("cpu")) for k, m in _models().items()}
    w, n = _waves()
    ni = {"src_tokens": w, "src_lengths": n}
    prev = torch.tensor([[2, 3], [2, 4], [2, 1]])
    calls = {
        "encoder.forward": lambda: ms["encoder"](**ni),
        "encdec.forward": lambda: ms["encdec"](**ni, prev_output_tokens=prev),
        "encdec.forward_encoder": lambda: ms["encdec"].forward_encoder(ni),
        "transducer.forward": lambda: ms["transducer"](**ni, prev_output_tokens=prev),
        "transducer.forward_encoder": lambda: ms["transducer"].forward_encoder(ni),
        "transducer greedy decoder": lambda: TransducerGreedyDecoder([ms["transducer"]], _Dict(), blank=0).decode(
            [ms["transducer"]], {"net_input": ni}),
        "transducer beam decoder": lambda: TransducerBeamSearchDecoder([ms["transducer"]], _Dict(), blank=0).decode(
            [ms["transducer"]], {"net_input": ni}),
    }
    for name, call in calls.items():
        with pytest.raises(RuntimeError, match=r"raw waveform input needs model\.frontend"):
            call()
