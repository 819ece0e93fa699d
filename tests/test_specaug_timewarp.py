"""CPU: adaptive SpecAugment with time warping, for precomputed features and raw waveforms.

tests/golden/specaug_timewarp.npz holds inputs, draws and outputs of the reference transform (with cv2's INTER_LINEAR
warp), written by oracle/pin_specaug.py.  The host draws must consume the NumPy RNG exactly like the reference, the
oracle and the per-op reference of esp_specaug_features (oracle/specaug.py) must reproduce its outputs, and a batch must
reach the encoder warped and masked through dataset -> collate -> model forward, with the per-op references standing in
for the CUDA ops."""
import json
import os
import wave

import numpy as np
import pytest
import torch

from oracle import ops_ref
from oracle import specaug as OS

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "specaug_timewarp.npz")
LIBRI_W5 = {"time_warp_W": 5, "freq_mask_F": 27, "freq_mask_N": 2, "time_mask_pm": 0.04, "time_mask_ps": 0.04}


def _cases():
    z = np.load(GOLDEN)
    for k, name in enumerate(z["names"].tolist()):
        warp = z["warp_%d" % k]
        yield dict(name=name, x=z["x_%d" % k], out=z["out_%d" % k], cfg=json.loads(str(z["cfg_%d" % k])),
                   seed=tuple(int(s) for s in z["seed_%d" % k]), warp=tuple(int(v) for v in warp[0]) if len(warp) else None,
                   fm=[tuple(int(v) for v in r) for r in z["fm_%d" % k]], tm=[tuple(int(v) for v in r) for r in z["tm_%d" % k]])


CASES = list(_cases())


def test_fixture_covers_the_warp_edges():
    by = {c["name"]: c for c in CASES}
    assert {c["cfg"]["time_warp_W"] for c in CASES} >= {0, 1, 5, 80}
    for W, m in ((5, 60), (80, 200)):
        assert by["W%d_w_max" % W]["warp"][1] == W - 1 and by["W%d_w_min" % W]["warp"][1] == -W + 1
        assert by["W%d_w_zero" % W]["warp"][1] == 0
        assert by["W%d_w0_min" % W]["warp"][0] == W and by["W%d_w0_max" % W]["warp"][0] == m - W - 1
        assert by["W%d_m_2W+1" % W]["warp"] is not None and by["W%d_m_2W" % W]["warp"] is None
    assert by["F83"]["x"].shape[1] == 83 and by["swbd"]["cfg"].get("time_mask_T") == 70
    assert by["F_below_mask_F"]["fm"] == [] and np.array_equal(by["F_below_mask_F"]["out"], by["F_below_mask_F"]["x"])


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_draws_consume_the_rng_like_the_reference(case):
    from espresso_b200.data import specaugment as SA

    cfg = SA.AdaptiveSpecAugmentConfig.from_config_dict(case["cfg"])
    m, F = case["x"].shape
    with SA.numpy_seed(*case["seed"]):
        warp, fm, tm = SA.draw_specaugment(cfg, m, F)
        after = np.random.randint(0, 2 ** 31 - 1)
    assert (warp, fm, tm) == (case["warp"], case["fm"], case["tm"])
    with SA.numpy_seed(*case["seed"]):
        OS.adaptive_specaugment(case["x"], **case["cfg"])
        assert np.random.randint(0, 2 ** 31 - 1) == after  # the oracle's stream, pinned against the reference's
    if cfg.time_warp_W == 0:  # draw_masks keeps its results for W = 0
        with SA.numpy_seed(*case["seed"]):
            assert SA.draw_masks(cfg, m, F) == (fm, tm)


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_matches_the_reference(case):
    with _seed(case["seed"]):
        got, warp, fm, tm = OS.adaptive_specaugment(case["x"], **case["cfg"])
    assert (warp, fm, tm) == (case["warp"], case["fm"], case["tm"])
    assert np.abs(got - case["out"]).max() <= 1e-6


def _seed(seed):
    from espresso_b200.data.specaugment import numpy_seed

    return numpy_seed(*seed)


@pytest.mark.parametrize("F", [80, 83, 40, 20])
def test_per_op_reference_matches_the_reference_on_ragged_batches(F):
    """oracle.specaug.specaug_features (the restatement the CUDA kernel is tested against) on the fixture's cases of one
    width packed into a right-padded batch, plus an utterance with no frames."""
    from espresso_b200.data import specaugment as SA

    cs = [c for c in CASES if c["x"].shape[1] == F]
    T = max(c["x"].shape[0] for c in cs) + 3
    x = torch.full((len(cs) + 1, T, F), 7.0)
    for b, c in enumerate(cs):
        x[b, :c["x"].shape[0]] = torch.from_numpy(c["x"])
    lens = torch.tensor([c["x"].shape[0] for c in cs] + [0], dtype=torch.int32)
    fm, tm = SA.pack_masks([c["fm"] for c in cs] + [[]], [c["tm"] for c in cs] + [[]])
    warp = torch.from_numpy(SA.pack_warps([c["warp"] for c in cs] + [None]))
    y = OS.specaug_features(x, lens, warp, torch.from_numpy(fm), torch.from_numpy(tm))
    for b, c in enumerate(cs):
        m = c["x"].shape[0]
        assert np.abs(y[b, :m].numpy() - c["out"]).max() <= 1e-6, c["name"]
        assert not y[b, m:].any()
    assert not y[-1].any()


def test_draw_masks_refuses_a_time_warp():
    from espresso_b200.data import specaugment as SA

    cfg = SA.AdaptiveSpecAugmentConfig.from_config_dict(LIBRI_W5)
    assert cfg.time_warp_W == 5
    for m in (0, 10, 100):
        with pytest.raises(ValueError, match="draw_specaugment"):
            SA.draw_masks(cfg, m, 80)
    with pytest.raises(ValueError):
        SA.AdaptiveSpecAugmentConfig.from_config_dict(dict(LIBRI_W5, time_warp_W=-1))


def test_items_and_batches_keep_their_keys_without_a_warp(tmp_path):
    from espresso_b200.data.asr_dataset import AudioFeatDataset
    from espresso_b200.data.collate import collate

    ids, rx, _ = _feats(tmp_path, 83)
    for W, has in ((0, False), (5, True)):
        ds = AudioFeatDataset(ids, rx, specaugment_config=dict(LIBRI_W5, time_warp_W=W), seed=3)
        it = ds[0]
        assert ("time_warp" in it) == has and set(it) - {"time_warp"} == {"source", "freq_masks", "time_masks"}
        b = collate([dict(ds[i], id=i) for i in range(len(ds))], 1, 2)
        assert ("time_warp" in b["net_input"]) == has
        assert set(b["net_input"]) - {"time_warp"} == {"src_tokens", "src_lengths", "freq_masks", "time_masks"}
        if has:
            tw = b["net_input"]["time_warp"]
            assert tw.dtype == torch.int32 and tuple(tw.shape) == (len(ds), 2)


def _feats(tmp_path, F):
    from espresso_b200.data.audio_io import write_kaldi_mat

    rs = np.random.RandomState(4)
    mats = [rs.randn(m, F).astype(np.float32) for m in (37, 61, 9, 48)]  # 9 <= 2W: no warp draw
    ark = str(tmp_path / "f.ark")
    rx = []
    with open(ark, "wb") as f:
        for i, mat in enumerate(mats):
            rx.append("%s:%d" % (ark, write_kaldi_mat(f, "u%d" % i, mat)))
    return ["u%d" % i for i in range(len(mats))], rx, mats


def _waves(tmp_path):
    rs = np.random.RandomState(5)
    ids, rx, waves = [], [], []
    for i, n in enumerate((9000, 5200, 1500, 7300)):
        x = rs.randint(-3000, 3000, size=n).astype(np.int16)
        p = str(tmp_path / ("w%d.wav" % i))
        with wave.open(p, "wb") as w:
            w.setnchannels(1)
            w.setsampwidth(2)
            w.setframerate(16000)
            w.writeframes(x.astype("<i2").tobytes())
        ids.append("w%d" % i)
        rx.append(p)
        waves.append(x.astype(np.float32))
    return ids, rx, waves


@pytest.fixture()
def cpu_ops(monkeypatch):
    from espresso_b200 import ops

    for name in dir(ops_ref):
        if name.startswith("_") or not callable(getattr(ops_ref, name)) or not hasattr(ops, name):
            continue
        monkeypatch.setattr(ops, name, getattr(ops_ref, name))
    monkeypatch.setattr(ops, "specaug_features", OS.specaug_features)
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


def _model(F):
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel

    class _Task:
        feat_dim, feat_in_channels, target_dictionary = F, 1, _Dict()

    cfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
        encoder=dict(embed_dim=32, ffn_embed_dim=64, layers=1, attention_heads=2, normalize_before=True,
                     relative_positional_embeddings=True, layer_type="transformer", conv_channels="[64, 64]",
                     conv_kernel_sizes="[(3, 3), (3, 3)]", conv_strides="[(2, 2), (2, 2)]")))
    torch.manual_seed(0)
    m = SpeechTransformerEncoderModel.build_model(cfg, _Task()).finalize_(torch.device("cpu"))
    seen = []
    enc_forward = m.encoder.forward
    m.encoder.forward = lambda x, lens, **kw: seen.append((x, lens)) or enc_forward(x, lens, **kw)
    return m, seen


@pytest.mark.parametrize("fmt", ["feat", "wave"])
def test_dataset_to_encoder_applies_warp_and_masks(cpu_ops, tmp_path, fmt):
    """The encoder receives, per utterance, what the reference's feature transform makes of the utterance under
    numpy_seed(seed, epoch, index): Kaldi features (83 wide) directly, waveforms after the fbank front end.  In eval mode
    the descriptors are ignored."""
    from espresso_b200.data.asr_dataset import AudioFeatDataset
    from espresso_b200.data.collate import collate
    from espresso_b200.data.frontend import OnTheFlyFbank
    from oracle import frontend as ofe

    if fmt == "feat":
        ids, rx, srcs = _feats(tmp_path, 83)
        ds = AudioFeatDataset(ids, rx, specaugment_config=LIBRI_W5, seed=3)
        plain = srcs
    else:
        ids, rx, srcs = _waves(tmp_path)
        ds = AudioFeatDataset(ids, rx, feat_dim=80, feature_type="fbank", specaugment_config=LIBRI_W5, seed=3)
        plain = [ofe.kaldi_fbank(w) for w in srcs]
    ds.set_epoch(2)
    items = [dict(ds[i], id=i) for i in range(len(ds))]
    assert sum(it["time_warp"] is not None for it in items) >= 2
    batch = collate(items, 1, 2)
    ni = batch["net_input"]
    model, seen = _model(plain[0].shape[1])
    if fmt == "wave":
        model.frontend = OnTheFlyFbank(None, None, out_dtype=torch.float32)
    model.train()
    with torch.no_grad():
        model(**ni)
    x, lens = seen[-1]
    assert x.dtype == torch.float32
    warped = 0
    for b, i in enumerate(batch["id"].tolist()):
        with _seed((3, 2, i)):
            want, warp, _, _ = OS.adaptive_specaugment(plain[i], **LIBRI_W5)
        m = want.shape[0]
        warped += warp is not None and warp[1] != 0
        assert int(lens[b]) == m
        assert np.abs(x[b, :m].numpy() - want).max() <= 1e-5, (fmt, i)
        assert not x[b, m:].any()
    assert warped >= 2
    model.eval()
    with torch.no_grad():
        model(**ni)
    x, _ = seen[-1]
    for b, i in enumerate(batch["id"].tolist()):
        assert np.abs(x[b, :plain[i].shape[0]].numpy() - plain[i]).max() <= (0 if fmt == "feat" else 1e-5)
