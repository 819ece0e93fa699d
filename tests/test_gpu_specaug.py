"""GPU: esp_specaug_features (adaptive SpecAugment with time warping on features) against the reference's outputs in
tests/golden/specaug_timewarp.npz (written by oracle/pin_specaug.py from the real transform and cv2), the waveform path
with a warp against the oracle front end, ragged batches with empty utterances, determinism, launch counts, and a
CUDA-graph replay of a feature-input training step."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "specaug_timewarp.npz")


def _cases():
    z = np.load(GOLDEN)
    out = []
    for k, name in enumerate(z["names"].tolist()):
        warp = z["warp_%d" % k]
        out.append(dict(name=name, x=z["x_%d" % k], out=z["out_%d" % k], cfg=json.loads(str(z["cfg_%d" % k])),
                        warp=tuple(int(v) for v in warp[0]) if len(warp) else None,
                        fm=[tuple(int(v) for v in r) for r in z["fm_%d" % k]],
                        tm=[tuple(int(v) for v in r) for r in z["tm_%d" % k]]))
    return out


def _batch(cs, pad_value=7.0, empty=True):
    """The cases packed into one right-padded batch [B, T, F] (padding filled with pad_value, which must not leak), plus
    an utterance with no frames."""
    from espresso_b200.data import specaugment as SA

    F = cs[0]["x"].shape[1]
    T = max(c["x"].shape[0] for c in cs) + 5
    n = len(cs) + int(empty)
    x = torch.full((n, T, F), pad_value)
    for b, c in enumerate(cs):
        x[b, :c["x"].shape[0]] = torch.from_numpy(c["x"])
    extra = [[]] * int(empty)
    lens = torch.tensor([c["x"].shape[0] for c in cs] + [0] * int(empty), dtype=torch.int32)
    fm, tm = SA.pack_masks([c["fm"] for c in cs] + extra, [c["tm"] for c in cs] + extra)
    warp = SA.pack_warps([c["warp"] for c in cs] + [None] * int(empty))
    return x, lens, torch.from_numpy(warp), torch.from_numpy(fm), torch.from_numpy(tm)


def _masked(c, m, F):
    """Boolean [m, F]: the elements the reference's masks cover."""
    sel = np.zeros((m, F), bool)
    for f0, f in c["fm"]:
        sel[:, f0:f0 + f] = True
    for t0, t in c["tm"]:
        sel[t0:t0 + t, :] = True
    return sel


def _bf16_ulp(v):
    a = np.maximum(np.abs(v), 2.0 ** -126)
    return 2.0 ** (np.floor(np.log2(a)) - 7)


@pytest.mark.parametrize("F", [80, 83, 40, 20])
@pytest.mark.parametrize("dt", ["f32", "bf16", "f32_to_bf16", "bf16_to_f32"])
def test_features_match_the_reference(F, dt):
    """fp32: within 1e-5 of the reference; bf16 output: within one bf16 ulp of it (the inputs are bf16 values, so every
    dtype sees the same numbers).  Masked elements hold one value, the utterance mean; padded frames are zero."""
    from espresso_b200 import ops

    cs = [c for c in _cases() if c["x"].shape[1] == F]
    x, lens, warp, fm, tm = _batch(cs)
    in_dt = torch.bfloat16 if dt.startswith("bf16") else torch.float32
    out_dt = torch.bfloat16 if dt.endswith("bf16") else torch.float32
    y = ops.specaug_features(x.to(DEV, in_dt), lens.to(DEV), warp.to(DEV), fm.to(DEV), tm.to(DEV), out_dtype=out_dt)
    assert y.dtype == out_dt and tuple(y.shape) == tuple(x.shape)
    y = y.float().cpu().numpy()
    for b, c in enumerate(cs):
        m = c["x"].shape[0]
        ref = c["out"]
        got = y[b, :m]
        err = np.abs(got - ref)
        if out_dt == torch.float32:
            assert err.max() <= 1e-5, (c["name"], float(err.max()))
        else:
            assert (err <= _bf16_ulp(ref)).all(), (c["name"], float(err.max()))
        sel = _masked(c, m, F)
        if sel.any():
            fill = got[sel][0]
            assert (got[sel] == fill).all(), c["name"]
            assert abs(fill - c["x"].astype(np.float64).mean()) <= (1e-6 if out_dt == torch.float32 else _bf16_ulp(fill))
        assert not y[b, m:].any(), c["name"]
    assert not y[-1].any()


def test_deterministic_and_launch_counts():
    """Same bits on every run (the mean is summed without atomics); 1 launch without masks, 2 with."""
    from espresso_b200 import lib, ops

    cs = [c for c in _cases() if c["x"].shape[1] == 80]
    x, lens, warp, fm, tm = (t.to(DEV) for t in _batch(cs))
    runs = []
    for _ in range(3):
        n0 = lib.launch_count()
        runs.append(ops.specaug_features(x, lens, warp, fm, tm))
        assert lib.launch_count() - n0 == 2
    assert all(torch.equal(runs[0], r) for r in runs[1:])
    n0 = lib.launch_count()
    y = ops.specaug_features(x, lens, warp)
    assert lib.launch_count() - n0 == 1
    n0 = lib.launch_count()
    y0 = ops.specaug_features(x, lens)
    assert lib.launch_count() - n0 == 1
    # without descriptors: a copy of the valid frames, zeros beyond
    valid = torch.arange(x.shape[1], device=DEV)[None, :] < lens[:, None].long()
    assert torch.equal(y0, torch.where(valid[..., None], x, torch.zeros_like(x)))
    # warp only: the warped frames the reference produces before masking, i.e. equal to the masked run off the masks
    z = runs[0].cpu().numpy()
    for b, c in enumerate(cs):
        m = c["x"].shape[0]
        keep = ~_masked(c, m, 80)
        assert np.array_equal(y[b, :m].cpu().numpy()[keep], z[b, :m][keep])


def test_host_refusals():
    from espresso_b200 import lib, ops

    x = torch.zeros(2, 10, 80, device=DEV)
    lens = torch.tensor([10, 4], dtype=torch.int32, device=DEV)
    too_many = torch.zeros(2, 65, 2, dtype=torch.int32, device=DEV)
    with pytest.raises(lib.EspressoB200Error, match="at most 64"):
        ops.specaug_features(x, lens, freq_masks=too_many)
    with pytest.raises(lib.EspressoB200Error):
        ops.specaug_features(x.cpu(), lens.cpu())


def test_waveform_path_with_a_warp_matches_the_oracle():
    """OnTheFlyFbank with a time warp (fused front end without masks into fp32, then esp_specaug_features) against the
    oracle front end + the reference transform with the same draws; ragged batch with an utterance shorter than one
    window.  bf16 output within the front end's 1e-3 log-mel bound plus one bf16 ulp."""
    from espresso_b200.data import specaugment as SA
    from espresso_b200.data.frontend import OnTheFlyFbank
    from oracle import frontend as ofe
    from oracle import specaug as OS

    cfg = {"time_warp_W": 5, "freq_mask_F": 27, "freq_mask_N": 2, "time_mask_pm": 0.04, "time_mask_ps": 0.04}
    sa = SA.AdaptiveSpecAugmentConfig.from_config_dict(cfg)
    waves = [ofe.synth_waveform(i, d) for i, d in enumerate([2.35, 1.0, 0.02, 3.17, 0.5])]
    N = max(len(w) for w in waves)
    wav = torch.zeros(len(waves), N)
    for b, w in enumerate(waves):
        wav[b, :len(w)] = torch.from_numpy(w)
    n = torch.tensor([len(w) for w in waves], dtype=torch.int32)
    draws, refs = [], []
    for i, w in enumerate(waves):
        fb = ofe.kaldi_fbank(w)
        with SA.numpy_seed(1, 1, i):
            draws.append(SA.draw_specaugment(sa, fb.shape[0], 80))
        if fb.shape[0] == 0:  # shorter than one window: no frames, nothing drawn
            refs.append(fb)
            continue
        with SA.numpy_seed(1, 1, i):
            refs.append(OS.adaptive_specaugment(fb, **cfg)[0])
    assert sum(d[0] is not None and d[0][1] != 0 for d in draws) >= 3
    fm, tm = SA.pack_masks([d[1] for d in draws], [d[2] for d in draws])
    tw = SA.pack_warps([d[0] for d in draws])
    for out_dt in (torch.float32, torch.bfloat16):
        fe = OnTheFlyFbank(None, None, out_dtype=out_dt)
        feats, lens = fe(wav.to(DEV), n.to(DEV), torch.from_numpy(fm).to(DEV), torch.from_numpy(tm).to(DEV),
                         time_warp=torch.from_numpy(tw).to(DEV))
        assert feats.dtype == out_dt
        feats = feats.float().cpu().numpy()
        for b, ref in enumerate(refs):
            m = ref.shape[0]
            assert int(lens[b]) == m
            tol = 1e-3 + (0 if out_dt == torch.float32 else _bf16_ulp(ref))
            assert (np.abs(feats[b, :m] - ref) <= tol).all(), (b, float(np.abs(feats[b, :m] - ref).max()))
            assert not feats[b, m:].any()


def test_graph_replay_of_a_feature_step_with_specaugment_equals_eager():
    """Trainer with CUDA graphs on feature batches carrying SpecAugment descriptors and time warps: the replayed step's
    encoder input is bit-identical to esp_specaug_features on the bucket-padded batch, and its gradients match the eager
    step's on that padded batch."""
    from espresso_b200 import ops
    from espresso_b200.criterions import CtcLossCriterion
    from espresso_b200.data import specaugment as SA
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel
    from espresso_b200.optim import NoamLRScheduler
    from espresso_b200.trainer import Trainer

    class _Dict:
        def __len__(self):
            return 50

        def pad(self):
            return 1

        def eos(self):
            return 2

        def index(self, sym):
            return 0

    class _Task:
        feat_dim, feat_in_channels, target_dictionary = 80, 1, _Dict()

    cfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, layernorm_embedding=True, max_source_positions=3600,
        encoder=dict(embed_dim=64, ffn_embed_dim=128, layers=2, attention_heads=4, normalize_before=True,
                     relative_positional_embeddings=True, layer_type="conformer", depthwise_conv_kernel_size=31)))
    torch.manual_seed(0)
    m = SpeechTransformerEncoderModel.build_model(cfg, _Task()).finalize_(DEV)
    seen = []
    enc_forward = m.encoder.forward
    m.encoder.forward = lambda x, lens, **kw: seen.append(x) or enc_forward(x, lens, **kw)
    pol = SA.AdaptiveSpecAugmentConfig.from_config_dict(
        {"time_warp_W": 5, "freq_mask_F": 27, "freq_mask_N": 2, "time_mask_pm": 0.04, "time_mask_ps": 0.04})

    def batch(T, lens, seed, U=6):
        rs = np.random.RandomState(seed)
        B = len(lens)
        feats = rs.randn(B, T, 80).astype(np.float32)
        draws = []
        for b, n in enumerate(lens):
            feats[b, n:] = 0
            with SA.numpy_seed(seed, 1, b):
                draws.append(SA.draw_specaugment(pol, n, 80))
        fm, tm = SA.pack_masks([d[1] for d in draws], [d[2] for d in draws])
        tgt = np.full((B, U + 1), 1, dtype=np.int64)
        for b in range(B):
            u = 2 + (b + seed) % (U - 1)
            tgt[b, :u] = rs.randint(4, 50, size=u)
            tgt[b, u] = 2
        lt = torch.tensor(lens)
        ni = {"src_tokens": torch.from_numpy(feats).to(DEV), "src_lengths": lt.to(DEV), "src_lengths_cpu": lt,
              "freq_masks": torch.from_numpy(fm).to(DEV), "time_masks": torch.from_numpy(tm).to(DEV),
              "time_warp": torch.from_numpy(SA.pack_warps([d[0] for d in draws])).to(DEV)}
        return {"net_input": ni, "target": torch.from_numpy(tgt).to(DEV)}

    crit = CtcLossCriterion(_Task())
    eager = Trainer(m, crit, NoamLRScheduler(0.0, 5, 64, 0.0), use_cuda_graphs=False)
    graphed = Trainer(m, crit, NoamLRScheduler(0.0, 5, 64, 0.0), use_cuda_graphs=True, bucket_frames=32, bucket_tokens=8)
    graphed._reduce_and_update = lambda: None  # keep the parameters fixed: compare raw gradient buffers
    # two buckets (4 or 8 time-mask slots), each seen first (eager), then captured, then replayed
    cases = [batch(128, [128, 90, 41], 1), batch(128, [120, 127, 64], 2), batch(117, [117, 60, 33], 3, U=5),
             batch(128, [128, 128, 100], 4), batch(100, [100, 99, 12], 5), batch(128, [128, 70, 50], 6),
             batch(110, [110, 80, 40], 7)]
    static_x = {}  # graph key -> the encoder input buffer of its capture, which every replay rewrites
    for i, smp in enumerate(cases):
        key, _ = graphed._signature(smp)
        n_seen = len(seen)
        graphed.train_step([smp])
        torch.cuda.synchronize()
        if len(seen) > n_seen:
            static_x[key] = seen[-1]
        got_x = static_x[key].clone()
        got = m.flat.g32.clone()
        ni, t = smp["net_input"], smp["target"]
        x = ni["src_tokens"]
        xp = torch.zeros(x.shape[0], 128, 80, device=DEV)
        xp[:, :x.shape[1]] = x
        pad4 = lambda d: torch.cat([d, torch.zeros(d.shape[0], (-d.shape[1]) % 4, 2, dtype=d.dtype, device=DEV)], 1)  # noqa: E731
        tp = torch.full((t.shape[0], 8), 1, dtype=t.dtype, device=DEV)
        tp[:, :t.shape[1]] = t
        padded = dict(ni, src_tokens=xp, freq_masks=pad4(ni["freq_masks"]), time_masks=pad4(ni["time_masks"]))
        want_x = ops.specaug_features(xp, ni["src_lengths"].to(torch.int32), ni["time_warp"], padded["freq_masks"],
                                      padded["time_masks"])
        assert torch.equal(got_x, want_x), i
        eager._fwd_bwd([{"net_input": padded, "target": tp}])
        torch.cuda.synchronize()
        ref = m.flat.g32.clone()
        denom = ref[: m.flat.numel].abs().max().item()
        err = (got - ref)[: m.flat.numel].abs().max().item() / denom
        assert err < 2e-2, (i, err)
    assert graphed.graph_hits >= 3 and len(graphed._graphs) == 2, (graphed.graph_hits, len(graphed._graphs))
