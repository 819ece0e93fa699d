"""CPU: encoders with absolute positions (relative positions off: the WSJ and Switchboard Transformer recipes) and relaxed
encoder-decoder attention.  The oracle (oracle/abspos.py) reproduces the fixtures recorded from the real reference
(tests/golden/encdec_transformer_abspos*.npz, encoder_conformer_abspos.npz: logits, losses, gradient sketches; the
parameters are oracle.abspos.seeded_state_dict); the host orchestration over the per-op reference (monkeypatched in for
the CUDA ops) reproduces the reference's logits and the oracle's gradients; the models refuse the configurations that are
not supported."""
import os

import numpy as np
import pytest
import torch

from oracle import abspos as OA
from oracle import decoder as OD
from oracle import ops_ref

V, PAD, EOS, BLANK = 50, 1, 2, 0
ENCDEC = ["encdec_transformer_abspos", "encdec_transformer_abspos_hd128"]


@pytest.fixture()
def cpu_ops(monkeypatch):
    from espresso_b200 import ops

    for name, fn in OA.cpu_ops().items():
        if hasattr(ops, name):
            monkeypatch.setattr(ops, name, fn)
    return ops


class _Dict:
    def __len__(self):
        return V

    def pad(self):
        return PAD

    def eos(self):
        return EOS

    def unk(self):
        return 3

    def index(self, sym):
        return 0


class _Task:
    feat_dim, feat_in_channels = 80, 1
    target_dictionary = _Dict()


def _load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name + ".npz"))


def _cfg(g, layer_type, **kw):
    from espresso_b200.models import SpeechTransformerConfig

    d, ffn, H, L = int(g["embed_dim"]), int(g["ffn_dim"]), int(g["heads"]), int(g["layers"])
    layers = dict(embed_dim=d, ffn_embed_dim=ffn, layers=L, attention_heads=H, normalize_before=True, learned_pos=False,
                  relative_positional_embeddings=False)
    return SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, max_source_positions=3600, max_target_positions=200,
        encoder=dict(layers, layer_type=layer_type, depthwise_conv_kernel_size=31),
        decoder=dict(layers, input_dim=d, output_dim=d, relaxed_attention_weight=float(g["relaxed"]) if "relaxed" in g else 0.0),
        **kw))


def _seeded(m, g):
    """The fixture's parameters: oracle.abspos.seeded_state_dict over the model's (= the reference's) keys and shapes."""
    m.load_state_dict(OA.seeded_state_dict({k: v.shape for k, v in m.state_dict().items()}, int(g["sd_seed"])), strict=True)
    return m


def build_encdec(g):
    from espresso_b200.models import SpeechTransformerModelBase

    return _seeded(SpeechTransformerModelBase.build_model(_cfg(g, "transformer"), _Task()), g)


def build_conformer(g):
    from espresso_b200.models import SpeechTransformerEncoderModel

    return _seeded(SpeechTransformerEncoderModel.build_model(_cfg(g, "conformer", layernorm_embedding=True), _Task()), g)


def encdec_criterion(g):
    from espresso_b200.criterions import LabelSmoothedCrossEntropyV2Criterion

    return LabelSmoothedCrossEntropyV2Criterion(_Task(), label_smoothing=float(g["eps"]), smoothing_type=str(g["smoothing"]))


def encdec_sample(g, dev=torch.device("cpu")):
    return {"net_input": {"src_tokens": torch.from_numpy(g["feats"]).to(dev), "src_lengths": torch.from_numpy(g["lens"]).to(dev),
                          "prev_output_tokens": torch.from_numpy(g["prev_output_tokens"]).to(dev)},
            "target": torch.from_numpy(g["target"]).to(dev)}


_BUFFER = ("running_", "num_batches_tracked", "_float_tensor", "version")


def oracle_sd(g, build, requires_grad=True, after=False):
    """The fixture's parameters as the oracle's fp32 state dict (parameters with requires_grad); after=True: with the
    BatchNorm running statistics the reference's training forward left (the eval pass's)."""
    keys = {k: v.shape for k, v in build(g).state_dict().items()}
    sd = OA.seeded_state_dict(keys, int(g["sd_seed"]))
    if after:
        sd.update({k[len("after."):]: torch.from_numpy(g[k]) for k in g.files if k.startswith("after.")})
    for k, v in sd.items():
        if requires_grad and v.is_floating_point() and not any(b in k for b in _BUFFER):
            v.requires_grad_(True)
    return sd


def _ecfg(g, layer_type):
    return dict(heads=int(g["heads"]), layers=int(g["layers"]), layer_type=layer_type, vocab=V if layer_type == "conformer" else None,
                layernorm_embedding=layer_type == "conformer", final_layer_norm=layer_type != "conformer")


def oracle_encdec(g, sd, training, relaxed=None):
    d, H, L = int(g["embed_dim"]), int(g["heads"]), int(g["layers"])
    dcfg = dict(dec_embed_dim=d, dec_heads=H, dec_layers=L, pad=PAD,
                relaxed_attention_weight=float(g["relaxed"]) if relaxed is None else relaxed)
    enc, _, pad = OA.encoder_forward(sd, _ecfg(g, "transformer"), torch.from_numpy(g["feats"]), torch.from_numpy(g["lens"]),
                                     training=training)
    return OA.decoder_forward(sd, dcfg, torch.from_numpy(g["prev_output_tokens"]), enc, pad if bool(pad.any()) else None,
                              training=training)


def oracle_encdec_train(g):
    """(logits, loss, nll, {name: fp32 gradient}) of the oracle's training step on the fixture."""
    sd = oracle_sd(g, build_encdec)
    logits = oracle_encdec(g, sd, training=True)
    loss, nll = OA.smoothed_ce(logits, torch.from_numpy(g["target"]), PAD, float(g["eps"]), str(g["smoothing"]), V)
    loss.backward()
    return logits.detach(), loss.item(), nll.item(), {k: v.grad for k, v in sd.items() if v.grad is not None}


def oracle_conformer_train(g):
    sd = oracle_sd(g, build_conformer)
    feats, lens, tgt = torch.from_numpy(g["feats"]), torch.from_numpy(g["lens"]), torch.from_numpy(g["target"])
    logits, ol, _ = OA.encoder_forward(sd, _ecfg(g, "conformer"), feats, lens, training=True)
    from oracle import conformer as OC

    loss = OC.ctc_criterion(logits, ol, tgt, PAD, EOS, BLANK)
    loss.backward()
    return logits.detach(), ol, loss.item(), {k: v.grad for k, v in sd.items() if v.grad is not None}


def grad_errors(ref_grads, grad_of):
    """Relative Frobenius error per parameter tensor against the oracle's fp32 gradients (analytically zero gradients
    skipped: rounding noise only), largest first."""
    out = []
    for name, ref in ref_grads.items():
        if OA.skip_grad(name):
            continue
        ref = ref.numpy()
        out.append((float(np.linalg.norm(grad_of(name) - ref) / max(np.linalg.norm(ref), 1e-3)), name))
    return sorted(out, reverse=True)


def sketch_errors(g, grads):
    return sorted(((OA.sketch_error(n, grads[n], g["gsk." + n]), n) for n in grads if not OA.skip_grad(n)), reverse=True)


# ---------------------------------------------------------------------------------------------------
# the oracle against the reference's recorded outputs
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ENCDEC)
def test_oracle_reproduces_encdec_fixture(name, golden_dir):
    g = _load(golden_dir, name)
    logits, loss, nll, grads = oracle_encdec_train(g)
    assert np.abs(logits.numpy() - g["logits"]).max() < 1e-5
    assert abs(loss - float(g["loss"])) < 1e-5 * float(g["loss"])
    assert abs(nll - float(g["nll"])) < 1e-5 * float(g["nll"])
    assert sorted(grads) == sorted(k[len("gsk."):] for k in g.files if k.startswith("gsk."))
    worst = sketch_errors(g, grads)
    assert worst[0][0] < 5e-5, worst[:4]
    # eval mode: no relaxation, BatchNorm running statistics as the training forward left them
    with torch.no_grad():
        ev = oracle_encdec(g, oracle_sd(g, build_encdec, requires_grad=False, after=True), training=False)
    assert np.abs(ev.numpy() - g["logits_eval"]).max() < 1e-5


def test_relaxation_changes_the_training_logits(golden_dir):
    """The WSJ-shaped fixture is only a test of relaxation if relaxation moves the logits."""
    g = _load(golden_dir, "encdec_transformer_abspos")
    assert float(g["relaxed"]) == 0.35
    sd = oracle_sd(g, build_encdec, requires_grad=False)
    with torch.no_grad():
        on = oracle_encdec(g, sd, training=True)
        off = oracle_encdec(g, sd, training=True, relaxed=0.0)
    assert (on - off).abs().max().item() > 1e-2


def test_oracle_reproduces_conformer_fixture(golden_dir):
    g = _load(golden_dir, "encoder_conformer_abspos")
    logits, ol, loss, grads = oracle_conformer_train(g)
    assert np.array_equal(ol.numpy(), g["out_lens"])
    assert np.abs(logits.numpy() - g["logits_train"]).max() < 1e-5
    assert abs(loss - float(g["loss_train"])) < 1e-5 * float(g["loss_train"])
    worst = sketch_errors(g, grads)
    assert worst[0][0] < 5e-5, worst[:4]


def test_abs_positions_rows():
    """Valid frame t reads row t + 1 of the padding_idx-0 table, padded frames the zero row; the native table is the
    same rows for every frame (padded rows are zeroed right after they are formed)."""
    from espresso_b200.modules.encoder_engine import sinusoidal_positions

    pad = torch.tensor([[False] * 5, [False] * 3 + [True] * 2])
    pe = OA.abs_positions(pad, 16)
    tab = OD.sinusoidal_table(6, 16, 0)
    assert torch.equal(pe[0], tab[1:6]) and torch.equal(pe[1, :3], tab[1:4]) and not pe[1, 3:].any()
    native = sinusoidal_positions(5, 16, 0, torch.device("cpu"), dtype=torch.float32)
    assert torch.equal(native, tab[1:6])


# ---------------------------------------------------------------------------------------------------
# the relaxed-attention backward: (1 - w) folded into the dq / dk GEMM alphas
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("drop_p", [0.0, 0.3])
def test_relaxed_attention_backward_matches_autograd(drop_p):
    """With g the dropout backward of dPd, dS = (1 - w) P (g - sum P g): the softmax backward on the PLAIN P, with the
    factor (1 - w) applied afterwards, equals autograd of the relaxed forward -- padded keys included (they carry w / Tk in
    the forward, but no gradient flows into the scores there)."""
    torch.manual_seed(0)
    H, B, Tq, Tk, w = 2, 3, 5, 11, 0.35
    ld = (Tk + 7) // 8 * 8
    lens = torch.tensor([11, 7, 4], dtype=torch.int32)
    s = torch.zeros(H, B, Tq, ld)
    s[..., :Tk] = torch.randn(H, B, Tq, Tk)
    s = s.to(torch.bfloat16)
    p, pd = OA.attn_softmax_relaxed_fwd(s, Tk, lens, w, drop_p, seed=9)
    assert not pd[..., Tk:].float().any()
    pad_cols = torch.arange(Tk)[None, :] >= lens[:, None].long()
    assert (pd.float()[..., :Tk][:, pad_cols[:, None, :].expand(B, Tq, Tk)] != 0).any() or drop_p > 0
    # autograd of the relaxed forward in fp32 on the same mask
    x = s.float()[..., :Tk].clone().requires_grad_(True)
    xm = x.masked_fill(pad_cols[None, :, None, :], float("-inf"))
    pr = torch.softmax(xm, dim=-1)
    keep = torch.ones(H, B, Tq, ld)
    if drop_p > 0:
        keep = ops_ref._drop(torch.ones(H, B, Tq, ld), drop_p, 9, ops_ref._flat_index(H, B, Tq, ld))
    relaxed = ((1 - w) * pr + w / Tk) * keep[..., :Tk]
    dpd = torch.randn(H, B, Tq, Tk)
    (relaxed * dpd).sum().backward()
    dpd_full = torch.zeros(H, B, Tq, ld)
    dpd_full[..., :Tk] = dpd
    ds, _ = ops_ref.attn_softmax_bwd(p, dpd_full.to(torch.bfloat16), Tk, 0, drop_p, 9, want_dbd=False)
    folded = (1 - w) * ds.float()[..., :Tk]
    ref = x.grad
    assert (folded - ref).abs().max().item() < 2e-2 * ref.abs().max().item()
    # exact in fp32: the factor commutes with the softmax backward
    exact = (1 - w) * (pr * (dpd * keep[..., :Tk] - (pr * dpd * keep[..., :Tk]).sum(-1, keepdim=True)))
    assert torch.allclose(exact, ref, atol=1e-6)


# ---------------------------------------------------------------------------------------------------
# the host orchestration over the per-op reference
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ENCDEC)
def test_encdec_state_dict_keys_match_reference(name, golden_dir):
    g = _load(golden_dir, name)
    keys = sorted(build_encdec(g).state_dict().keys())
    assert keys == sorted(str(k) for k in g["state_dict_keys"])
    assert "encoder.embed_positions._float_tensor" in keys
    assert not any("pos_bias" in k or "pos_proj" in k or "positional_embedding" in k for k in keys)


def test_conformer_state_dict_keys_match_reference(golden_dir):
    g = _load(golden_dir, "encoder_conformer_abspos")
    keys = sorted(build_conformer(g).state_dict().keys())
    assert keys == sorted(str(k) for k in g["state_dict_keys"])
    assert "encoder.embed_positions._float_tensor" in keys


@pytest.mark.parametrize("name", ENCDEC)
def test_encdec_host_path_vs_reference_fixture(name, golden_dir, cpu_ops):
    g = _load(golden_dir, name)
    _, _, _, ref_grads = oracle_encdec_train(g)
    m = build_encdec(g).finalize_(torch.device("cpu"))
    crit = encdec_criterion(g)
    sample = encdec_sample(g)
    m.train()
    m.flat.zero_grad()
    loss, sample_size, log = crit(m, sample)
    assert abs(loss.item() - float(g["loss"])) < 5e-3 * float(g["loss"])
    assert abs(log["nll_loss"].item() - float(g["nll"])) < 5e-3 * float(g["nll"])
    loss.backward()
    m.encoder.sync_torch_grads_()
    worst = grad_errors(ref_grads, lambda n: m.flat.grad(n).numpy())
    print(name, worst[:6])
    assert worst[0][0] < 0.25, worst[:5]
    assert max(w_ for w_, n in worst if "pre_encoder" not in n) < 0.1, worst[:8]
    assert np.median([w_ for w_, _ in worst]) < 0.03
    # eval first: the fixture's eval pass saw the BatchNorm running statistics of ONE training forward
    for mode, key in (("eval", "logits_eval"), ("train", "logits")):  # train: relaxation on, as in the training forward
        m.train(mode == "train")
        with torch.no_grad():
            logits, _ = m(**sample["net_input"])
        assert np.abs(logits.float().numpy() - g[key]).max() < 2e-2 * np.ptp(g[key]), mode


def test_conformer_host_path_vs_reference_fixture(golden_dir, cpu_ops):
    from espresso_b200.criterions import CtcLossCriterion

    g = _load(golden_dir, "encoder_conformer_abspos")
    _, _, _, ref_grads = oracle_conformer_train(g)
    m = build_conformer(g).finalize_(torch.device("cpu"))
    crit = CtcLossCriterion(_Task(), zero_infinity=True, sentence_avg=True)
    sample = {"net_input": {"src_tokens": torch.from_numpy(g["feats"]), "src_lengths": torch.from_numpy(g["lens"])},
              "target": torch.from_numpy(g["target"]), "ntokens": 13}
    m.train()
    m.flat.zero_grad()
    loss, _, _ = crit(m, sample)
    assert abs(loss.item() - float(g["loss_train"])) < 5e-3 * float(g["loss_train"])
    loss.backward()
    m.encoder.sync_torch_grads_()
    worst = grad_errors(ref_grads, lambda n: m.flat.grad(n).numpy())
    print(worst[:6])
    assert worst[0][0] < 0.25, worst[:5]
    assert max(w_ for w_, n in worst if "pre_encoder" not in n) < 0.1, worst[:8]
    assert np.median([w_ for w_, _ in worst]) < 0.03
    m.eval()
    with torch.no_grad():
        net = m(**sample["net_input"])
    logits = net["encoder_out"][0].transpose(0, 1).float().numpy()
    assert np.abs(logits - g["logits_eval"]).max() < 2e-2 * np.ptp(g["logits_eval"])


# ---------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------
def test_learned_absolute_encoder_positions_are_refused(golden_dir):
    from espresso_b200.models import SpeechTransformerEncoderModel

    cfg = _cfg(_load(golden_dir, "encoder_conformer_abspos"), "transformer")
    cfg.encoder.learned_pos = True
    with pytest.raises(NotImplementedError, match="learned absolute"):
        SpeechTransformerEncoderModel.build_model(cfg, _Task())


def test_relaxed_attention_with_scheduled_sampling_is_refused(golden_dir):
    from espresso_b200.models import SpeechTransformerModelBase

    cfg = _cfg(_load(golden_dir, "encdec_transformer_abspos"), "transformer")
    cfg.scheduled_sampling_probs = (0.9,)
    with pytest.raises(NotImplementedError, match="scheduled sampling"):
        SpeechTransformerModelBase.build_model(cfg, _Task())
    cfg.decoder.relaxed_attention_weight = 0.0
    SpeechTransformerModelBase.build_model(cfg, _Task())  # scheduled sampling alone stays supported
