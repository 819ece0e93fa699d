"""CPU: which attention kernels the encoder's self-attention runs, per position source, head dim and length.

The choice comes from shapes alone: head dim 64 runs the fused forward and backward (csrc/attn_fused.cu,
csrc/attn_fused_bwd.cu), any other head dim the unfused chain (score GEMM, softmax, P v GEMM; with relative positions
also the BD GEMM added to the scores in skewed layout).  With relative positions the fused backward writes the skewed
score gradient through a kernel that takes rows of at most 1024 keys, so longer inputs take the unfused backward
after the fused forward.  The engine runs on the per-op reference (oracle/ops_ref.py, oracle/abspos.py), and a spy
counts the calls."""
import inspect

import pytest
import torch

from oracle import abspos as OA
from oracle import ops_ref


@pytest.fixture()
def calls(monkeypatch):
    """Installs the per-op reference for espresso_b200.ops; returns the list of (name, bound arguments) it receives."""
    from espresso_b200 import ops

    seen = []

    def spy(name, fn, sig):
        def call(*a, **kw):
            b = sig.bind(*a, **kw)
            b.apply_defaults()
            seen.append((name, dict(b.arguments)))
            return fn(*a, **kw)
        return call

    for name, fn in OA.cpu_ops().items():
        if hasattr(ops, name):
            monkeypatch.setattr(ops, name, spy(name, fn, inspect.signature(getattr(ops, name))))
    ops_ref.set_seed_tensor(None)
    return seen


class _Dict:
    def __len__(self):
        return 20

    def pad(self):
        return 1

    def eos(self):
        return 2

    def index(self, sym):
        return 0


class _Task:
    feat_dim, feat_in_channels = 80, 1
    target_dictionary = _Dict()


def _engine(pos, hd, H=1, layer_type="transformer"):
    """One-layer encoder with heads of width hd; pos: "sinusoidal" | "learned" (width d) | "learned_shared" (width
    head_dim, shared across heads) relative positions, or "absolute"."""
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel

    enc = dict(embed_dim=H * hd, ffn_embed_dim=32, layers=1, attention_heads=H, normalize_before=True,
               learned_pos=pos.startswith("learned"), relative_positional_embeddings=pos != "absolute",
               share_learned_relative_positional_embeddings_across_heads=pos == "learned_shared",
               layer_type=layer_type, depthwise_conv_kernel_size=5)
    cfg = SpeechTransformerConfig.from_dict(dict(dropout=0.1, attention_dropout=0.1, activation_dropout=0.1,
                                                 max_source_positions=3600, encoder=enc))
    m = SpeechTransformerEncoderModel.build_model(cfg, _Task())
    m.load_state_dict(OA.seeded_state_dict({k: v.shape for k, v in m.state_dict().items()}, 5), strict=True)
    m.finalize_(torch.device("cpu"))
    eng = m.encoder.engine
    eng.training, eng.seed = True, 3
    return eng


def _step(eng, T, B=2):
    g = torch.Generator().manual_seed(0)
    xc = torch.randn(B, T, eng.P("fc0.weight").shape[1], generator=g).to(torch.bfloat16)
    lens = torch.tensor([T] + [T - 3] * (B - 1), dtype=torch.int32)
    out = eng.forward(xc, lens, True)
    eng.backward((0.1 * torch.randn(out.shape, generator=g)).to(torch.bfloat16))


def _plan(calls):
    def n(name, pred=lambda a: True):
        return sum(1 for c, a in calls if c == name and pred(a))

    return dict(fused_fwd=n("attn_fused_fwd"), fused_bwd=n("attn_fused_bwd"),
                fused_bwd_dbd=n("attn_fused_bwd", lambda a: a["ldp"] is not None),
                softmax_fwd=n("attn_softmax_fwd"), softmax_bwd=n("attn_softmax_bwd", lambda a: not a["want_dbd"]),
                softmax_bwd_dbd=n("attn_softmax_bwd", lambda a: a["want_dbd"]),
                skew_gemm=n("gemm", lambda a: a["skew_r"] > 0))


_NONE = dict(fused_fwd=0, fused_bwd=0, fused_bwd_dbd=0, softmax_fwd=0, softmax_bwd=0, softmax_bwd_dbd=0, skew_gemm=0)
RELATIVE = ["sinusoidal", "learned", "learned_shared"]


@pytest.mark.parametrize("pos", RELATIVE + ["absolute"])
def test_head_dim_64_runs_the_fused_kernels_both_ways(pos, calls):
    _step(_engine(pos, 64, H=2), 12)
    dbd = int(pos != "absolute")  # the skewed copy of dS only serves relative positions
    assert _plan(calls) == dict(_NONE, fused_fwd=1, fused_bwd=1, fused_bwd_dbd=dbd)


@pytest.mark.parametrize("hd", [16, 128])
@pytest.mark.parametrize("pos", RELATIVE + ["absolute"])
def test_other_head_dims_run_the_unfused_chain_both_ways(pos, hd, calls):
    _step(_engine(pos, hd, H=2), 12)
    if pos == "absolute":
        assert _plan(calls) == dict(_NONE, softmax_fwd=1, softmax_bwd=1)
    else:
        assert _plan(calls) == dict(_NONE, softmax_fwd=1, softmax_bwd_dbd=1, skew_gemm=1)


@pytest.mark.parametrize("pos", ["sinusoidal", "learned_shared"])
def test_relative_positions_above_1024_frames_take_the_unfused_backward(pos, calls):
    _step(_engine(pos, 64), 1025)
    assert _plan(calls) == dict(_NONE, fused_fwd=1, softmax_bwd_dbd=1)


def test_absolute_positions_above_1024_frames_stay_fused(calls):
    _step(_engine("absolute", 64), 1025)
    assert _plan(calls) == dict(_NONE, fused_fwd=1, fused_bwd=1)


@pytest.mark.parametrize("pos", ["sinusoidal", "absolute"])
def test_attention_masks_off_the_fused_kernel_are_refused(pos, calls):
    eng = _engine(pos, 16, H=2, layer_type="conformer")
    T = 12
    eng.key_bounds = (torch.zeros(T, dtype=torch.int32), torch.full((T,), T, dtype=torch.int32))
    with pytest.raises(NotImplementedError, match="head_dim 64"):
        _step(eng, T)
    assert _plan(calls) == _NONE
