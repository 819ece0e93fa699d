"""GPU: attention without positions (absolute-position encoders: the WSJ and Switchboard Transformer recipes) and relaxed
encoder-decoder attention on the sm_90a kernels.

  * the fused forward without positions (esp_attn_fused_fwd with pos == NULL) is bit-identical to the relative-position
    kernel given an all-zero position table -- S + bf16(0) is exact in fp32, so any difference is a bug;
  * the fused backward with dbd == NULL writes the same dS / dK / dV as the relative-position call and nothing else, and
    runs beyond the skew kernel's 1024 frames;
  * esp_attn_softmax_relaxed_fwd against its per-op statement (oracle/abspos.py);
  * the three models against the fixtures recorded from the real reference, a CUDA-graph replay of the WSJ-shaped step,
    search against the host path, and the launches the variant saves per layer."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_attn_fwd_bitexact import CASES  # noqa: E402  (the shape list of the rel-pos bit-exact test)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _no_device_seed():
    from espresso_b200 import ops

    ops.set_seed_tensor(None)
    yield
    ops.set_seed_tensor(None)


def _inputs(name):
    """The bit-exact test's inputs for case `name` (CPU generators)."""
    from espresso_b200.tools.utils import chunk_streaming_bounds

    B, T, H, lens, kb, shared, drop, dseed, save = CASES[name]
    d = H * 64
    g = torch.Generator(device="cpu").manual_seed(1000 * T + B)
    qkv = (torch.randn(B * T, 3 * d, generator=g) * 0.7).bfloat16().to(DEV)
    qu = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16().to(DEV)
    lens_t = None
    if lens == "ragged":
        ln = torch.randint(max(1, T // 3), T + 1, (B,), generator=g, dtype=torch.int32)
        ln[0] = T
        lens_t = ln.to(DEV)
    bounds = None
    if kb is not None:
        lo, hi = chunk_streaming_bounds(T, *kb, always_partial_in_last=True)
        bounds = (torch.from_numpy(lo.astype(np.int32)).to(DEV), torch.from_numpy(hi.astype(np.int32)).to(DEV))
    return B, T, H, d, qkv, qu, lens_t, bounds, drop, dseed, save


def _device_seed(dseed):
    from espresso_b200 import ops

    ops.set_seed_tensor(None if dseed is None else
                        torch.tensor([dseed - 2 ** 64 if dseed >= 2 ** 63 else dseed], dtype=torch.int64, device=DEV))


@pytest.mark.parametrize("name", sorted(CASES))
def test_fwd_without_positions_equals_zero_table_bitwise(name):
    from espresso_b200 import ops

    B, T, H, d, qkv, qu, lens_t, bounds, drop, dseed, save = _inputs(name)
    zeros = torch.zeros(2 * T - 1, 64, dtype=torch.bfloat16, device=DEV)
    k, v = qkv[:, d:2 * d], qkv[:, 2 * d:]
    _device_seed(dseed)
    ref = ops.attn_fused_fwd(qu, qu, k, v, zeros, B, T, H, lens_t, drop_p=drop, seed=777, save_probs=save, pos_hstride=0,
                             key_bounds=bounds)
    got = ops.attn_fused_fwd(qu, None, k, v, None, B, T, H, lens_t, drop_p=drop, seed=777, save_probs=save, key_bounds=bounds)
    torch.cuda.synchronize()
    for what, a, b in zip(("ctx", "P", "Pd"), got, ref):
        assert (a is None) == (b is None), what
        if a is not None:  # the whole buffers: padding columns [T, ld) included
            assert torch.equal(a.view(torch.int16), b.view(torch.int16)), (name, what)


@pytest.mark.parametrize("T,drop", [(1, 0.0), (129, 0.0), (300, 0.1), (754, 0.1)])
def test_bwd_without_skew_equals_rel_pos_call_and_writes_nothing_else(T, drop):
    from espresso_b200 import ops

    B, H = 3, 4
    d = H * 64
    g = torch.Generator(device="cpu").manual_seed(T)
    qkv = (torch.randn(B * T, 3 * d, generator=g) * 0.7).bfloat16().to(DEV)
    qu = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16().to(DEV)
    dctx = (torch.randn(B * T, d, generator=g) * 0.5).bfloat16().to(DEV)
    lens = torch.tensor([T, max(1, T // 2), max(1, T // 3)], dtype=torch.int32, device=DEV)
    k, v = qkv[:, d:2 * d], qkv[:, 2 * d:]
    ctx, p, pd = ops.attn_fused_fwd(qu, None, k, v, None, B, T, H, lens, drop_p=drop, seed=5)
    ldp = (2 * T - 1 + 7) // 8 * 8
    sentinel = -12345.0
    out = []
    for with_skew in (True, False):
        dqkv = torch.full((B * T, 3 * d), sentinel, dtype=torch.bfloat16, device=DEV)
        ds, dbd = ops.attn_fused_bwd(dctx, ctx, qu, v, p, pd, B, T, H, ldp if with_skew else None, dqkv[:, d:2 * d],
                                     dqkv[:, 2 * d:], drop_p=drop, seed=5)
        torch.cuda.synchronize()
        assert (dbd is None) == (not with_skew)
        assert (dqkv[:, :d] == sentinel).all()  # the dq columns are not touched
        out.append((ds, dqkv))
    (ds1, dqkv1), (ds0, dqkv0) = out
    assert torch.equal(ds0.view(torch.int16), ds1.view(torch.int16))
    assert torch.equal(dqkv0.view(torch.int16), dqkv1.view(torch.int16))


def test_bwd_without_skew_beyond_1024_frames_vs_ops_ref():
    from espresso_b200 import ops
    from oracle import abspos as OA

    B, H, T = 2, 2, 1100
    d = H * 64
    g = torch.Generator(device="cpu").manual_seed(11)
    qkv = (torch.randn(B * T, 3 * d, generator=g) * 0.7).bfloat16()
    qu = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16()
    dctx = (torch.randn(B * T, d, generator=g) * 0.5).bfloat16()
    lens = torch.tensor([T, 1031], dtype=torch.int32)
    k, v = qkv[:, d:2 * d], qkv[:, 2 * d:]
    ctx, p, pd = ops.attn_fused_fwd(qu.to(DEV), None, k.to(DEV), v.to(DEV), None, B, T, H, lens.to(DEV), seed=3)
    rctx, rp, rpd = OA.attn_fused_fwd(qu, None, k, v, None, B, T, H, lens)
    assert (ctx.cpu().float() - rctx.float()).abs().max().item() < 2e-2 * rctx.float().abs().max().item()
    dqkv = torch.zeros(B * T, 3 * d, dtype=torch.bfloat16, device=DEV)
    ds, dbd = ops.attn_fused_bwd(dctx.to(DEV), ctx, qu.to(DEV), v.to(DEV), p, pd, B, T, H, None, dqkv[:, d:2 * d],
                                 dqkv[:, 2 * d:])
    rdqkv = torch.zeros(B * T, 3 * d, dtype=torch.bfloat16)
    rds, _ = OA.attn_fused_bwd(dctx, ctx.cpu(), qu, v, p.cpu(), pd.cpu(), B, T, H, None, rdqkv[:, d:2 * d], rdqkv[:, 2 * d:])
    torch.cuda.synchronize()
    assert dbd is None
    for a, b in ((ds.cpu(), rds), (dqkv.cpu()[:, d:], rdqkv[:, d:])):
        err = (a.float() - b.float()).norm() / b.float().norm()
        assert err < 1e-2, err


@pytest.mark.parametrize("Tk,drop,dseed", [(37, 0.0, None), (37, 0.2, None), (300, 0.1, 77), (1000, 0.1, None)])
def test_relaxed_softmax_vs_ops_ref(Tk, drop, dseed):
    from espresso_b200 import ops
    from oracle import abspos as OA
    from oracle import ops_ref

    H, B, Tq, w = 2, 3, 9, 0.35
    ld = (Tk + 7) // 8 * 8
    g = torch.Generator(device="cpu").manual_seed(Tk)
    s = torch.zeros(H, B, Tq, ld)
    s[..., :Tk] = torch.randn(H, B, Tq, Tk, generator=g) * 3
    s = s.bfloat16()
    lens = torch.tensor([Tk, Tk // 2, 3], dtype=torch.int32)
    _device_seed(dseed)
    ops_ref.set_seed_tensor(None if dseed is None else torch.tensor([dseed]))
    try:
        p, pd = ops.attn_softmax_relaxed_fwd(s.to(DEV), Tk, lens.to(DEV), w, drop_p=drop, seed=21)
        rp, rpd = OA.attn_softmax_relaxed_fwd(s, Tk, lens, w, drop_p=drop, seed=21)
    finally:
        ops_ref.set_seed_tensor(None)
    p, pd = p.cpu().float(), pd.cpu().float()
    rp, rpd = rp.float(), rpd.float()
    assert (p - rp).abs().max().item() < 1e-2
    assert (pd - rpd).abs().max().item() < 2e-2
    assert torch.equal(pd == 0, rpd == 0)  # the dropout masks (kept relaxed values are > 0)
    assert not pd[..., Tk:].any() and not p[..., Tk:].any()
    # padded keys carry w / Tk (scaled where kept): exactly the reference's bf16 value
    add = torch.tensor(np.float32(w / Tk)).bfloat16().float()
    for b, n in enumerate(lens.tolist()):
        cols = pd[:, b, :, n:Tk]
        if drop == 0:
            assert torch.equal(cols, add.expand_as(cols))
        assert torch.equal(cols, rpd[:, b, :, n:Tk])


# ---------------------------------------------------------------------------------------------------
# models against the reference fixtures
# ---------------------------------------------------------------------------------------------------
def _gpu_grad_bounds(worst):
    med = float(np.median([w for w, _ in worst]))
    inner = max(w for w, n in worst if "pre_encoder" not in n)
    return med, inner


@pytest.mark.parametrize("name", ["encdec_transformer_abspos", "encdec_transformer_abspos_hd128"])
def test_encdec_vs_reference_fixture(name, golden_dir, parity):
    import test_abspos_host as HH

    g = HH._load(golden_dir, name)
    _, _, _, ref_grads = HH.oracle_encdec_train(g)  # the oracle's fp32 gradients (pinned to the reference's sketches)
    m = HH.build_encdec(g).finalize_(DEV)
    crit = HH.encdec_criterion(g)
    sample = HH.encdec_sample(g, DEV)
    m.train()
    m.flat.zero_grad()
    loss, _, log = crit(m, sample)
    loss.backward()
    m.encoder.sync_torch_grads_()
    torch.cuda.synchronize()
    parity("%s: loss relative" % name, abs(loss.item() - float(g["loss"])) / float(g["loss"]), 5e-3)
    parity("%s: nll relative" % name, abs(log["nll_loss"].item() - float(g["nll"])) / float(g["nll"]), 5e-3)
    worst = HH.grad_errors(ref_grads, lambda n: m.flat.grad(n).cpu().numpy())
    med, inner = _gpu_grad_bounds(worst)
    print(name, worst[:6])
    parity("%s: median gradient rel-Frobenius" % name, med, 0.03)
    parity("%s: worst gradient rel-Frobenius (outside the conv front)" % name, inner, 0.1)
    parity("%s: worst gradient rel-Frobenius" % name, worst[0][0], 0.25)
    # eval first: the fixture's eval pass saw the BatchNorm running statistics of ONE training forward
    for mode, key in (("eval", "logits_eval"), ("train", "logits")):
        m.train(mode == "train")
        with torch.no_grad():
            logits, _ = m(**sample["net_input"])
        ours, ref = logits.float().cpu().numpy(), g[key]
        parity("%s: %s logits max error / range" % (name, mode), np.abs(ours - ref).max() / np.ptp(ref), 2e-2)
        parity("%s: %s logits rel-Frobenius" % (name, mode), np.linalg.norm(ours - ref) / np.linalg.norm(ref), 1.5e-2)


def test_conformer_ctc_vs_reference_fixture(golden_dir, parity):
    import test_abspos_host as HH
    from espresso_b200.criterions import CtcLossCriterion

    g = HH._load(golden_dir, "encoder_conformer_abspos")
    _, _, _, ref_grads = HH.oracle_conformer_train(g)
    m = HH.build_conformer(g).finalize_(DEV)
    crit = CtcLossCriterion(HH._Task(), zero_infinity=True, sentence_avg=True)
    sample = {"net_input": {"src_tokens": torch.from_numpy(g["feats"]).to(DEV), "src_lengths": torch.from_numpy(g["lens"]).to(DEV)},
              "target": torch.from_numpy(g["target"]).to(DEV), "ntokens": 13}
    m.train()
    m.flat.zero_grad()
    loss, _, _ = crit(m, sample)
    loss.backward()
    m.encoder.sync_torch_grads_()
    torch.cuda.synchronize()
    tag = "encoder_conformer_abspos"
    parity("%s: loss relative" % tag, abs(loss.item() - float(g["loss_train"])) / float(g["loss_train"]), 5e-3)
    worst = HH.grad_errors(ref_grads, lambda n: m.flat.grad(n).cpu().numpy())
    med, inner = _gpu_grad_bounds(worst)
    print(tag, worst[:6])
    parity("%s: median gradient rel-Frobenius" % tag, med, 0.03)
    parity("%s: worst gradient rel-Frobenius (outside the conv front)" % tag, inner, 0.1)
    parity("%s: worst gradient rel-Frobenius" % tag, worst[0][0], 0.25)
    m.eval()
    with torch.no_grad():
        net = m(**sample["net_input"])
    ours, ref = net["encoder_out"][0].transpose(0, 1).float().cpu().numpy(), g["logits_eval"]
    parity("%s: eval logits max error / range" % tag, np.abs(ours - ref).max() / np.ptp(ref), 2e-2)
    parity("%s: eval logits rel-Frobenius" % tag, np.linalg.norm(ours - ref) / np.linalg.norm(ref), 1.5e-2)


def test_graph_replay_of_wsj_step_equals_eager(golden_dir):
    """The WSJ-shaped training step (relaxed encoder attention) replayed from a CUDA graph == the eager step.  The buckets
    equal the batch's shape here; with larger buckets relaxation divides by the bucketed key count, as the reference would
    under pad_to_multiple."""
    import test_abspos_host as HH
    from espresso_b200.optim import NoamLRScheduler
    from espresso_b200.trainer import Trainer

    g = HH._load(golden_dir, "encdec_transformer_abspos")
    m = HH.build_encdec(g).finalize_(DEV)
    sample = HH.encdec_sample(g, DEV)
    sample["net_input"]["src_lengths_cpu"] = torch.from_numpy(g["lens"])
    sample["net_input"]["prev_output_tokens_cpu"] = torch.from_numpy(g["prev_output_tokens"])
    tr = Trainer(m, HH.encdec_criterion(g), NoamLRScheduler(0.0, 5, 64, 0.0), use_cuda_graphs=True,
                 bucket_frames=g["feats"].shape[1], bucket_tokens=g["target"].shape[1])
    tr._reduce_and_update = lambda: None  # keep the parameters fixed: compare raw gradient buffers
    n = m.flat.numel
    tr.train_step([sample])  # eager
    tr.train_step([sample])  # capture + replay
    torch.cuda.synchronize()
    assert len(tr._graphs) == 1
    g_graph = m.flat.g32[:n].clone()
    tr._fwd_bwd([sample])
    torch.cuda.synchronize()
    g_eager = m.flat.g32[:n].clone()
    err = (g_graph - g_eager).abs().max().item() / g_eager.abs().max().item()
    assert err < 2e-2, err


def test_beam_search_matches_host_path(golden_dir, monkeypatch):
    import test_abspos_host as HH
    from espresso_b200 import ops
    from espresso_b200.sequence_generator import SequenceGenerator
    from oracle import abspos as OA

    g = HH._load(golden_dir, "encdec_transformer_abspos")
    feats, lens = torch.from_numpy(g["feats"]), torch.from_numpy(g["lens"])
    # beam 1: where the two searches part, the step's decision is a single arg-max, which the host model can score
    kw = dict(beam_size=1, max_len_a=0.0, max_len_b=10)
    m = HH.build_encdec(g).finalize_(DEV)
    m.eval()
    gpu = SequenceGenerator([m], HH._Dict(), **kw).generate(
        [m], {"net_input": {"src_tokens": feats.to(DEV), "src_lengths": lens.to(DEV)}})
    for name, fn in OA.cpu_ops().items():
        if hasattr(ops, name):
            monkeypatch.setattr(ops, name, fn)
    mh = HH.build_encdec(g).finalize_(torch.device("cpu"))
    mh.eval()
    host = SequenceGenerator([mh], HH._Dict(), **kw).generate([mh], {"net_input": {"src_tokens": feats, "src_lengths": lens}})
    assert len(gpu) == len(host) == feats.shape[0]
    same = 0
    for b, (a, h) in enumerate(zip(gpu, host)):
        ta, th = a[0]["tokens"].cpu().tolist(), h[0]["tokens"].tolist()
        if ta == th:
            same += 1
            continue
        # the first step where they part must be a near-tie of the host model: its log-probabilities of the two tokens,
        # after the common prefix, within the bf16 logit error of the device path (logits within 0.5 % of their range)
        i = next(k for k in range(min(len(ta), len(th))) if ta[k] != th[k])
        prev = torch.tensor([HH.EOS] + th[:i])[None]
        with torch.no_grad():
            logits, _ = mh(feats[b:b + 1], lens[b:b + 1], prev)
        lp = torch.log_softmax(logits[0, -1].float(), dim=-1)
        gap = (lp[th[i]] - lp[ta[i]]).item()
        print("sentence %d parts at step %d: device %d, host %d, host log-prob gap %.4f" % (b, i, ta[i], th[i], gap))
        assert 0.0 <= gap < 0.05, (b, i, ta, th, gap)
    assert same >= 1, "no sentence decoded identically"


def test_launches_saved_per_layer():
    """A training step of an absolute-position Transformer layer launches 8 kernels fewer than the relative-position
    layer of the same shape (head dim 64, fused kernels):
      forward   pos_proj GEMM                                                                          1
      backward  skew copy of dS, dq_v GEMM, dpos GEMM, qprep_bwd, pos_proj weight gradient, two colsums   7
    Everything else (layer norms, projections, the fused attention forward and score-side backward, dq = s dS k in place
    of dq_u) is launched by both."""
    from espresso_b200 import lib
    from espresso_b200.criterions import CtcLossCriterion
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel

    import test_abspos_host as HH

    L = 2
    counts = {}
    for rel in (True, False):
        cfg = SpeechTransformerConfig.from_dict(dict(
            dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, max_source_positions=3600,
            encoder=dict(embed_dim=128, ffn_embed_dim=256, layers=L, attention_heads=2, normalize_before=True,
                         learned_pos=False, relative_positional_embeddings=rel, layer_type="transformer")))
        torch.manual_seed(0)
        m = SpeechTransformerEncoderModel.build_model(cfg, HH._Task()).finalize_(DEV)
        crit = CtcLossCriterion(HH._Task(), zero_infinity=True)
        rs = np.random.RandomState(0)
        sample = {"net_input": {"src_tokens": torch.from_numpy(rs.randn(2, 200, 80).astype(np.float32)).to(DEV),
                                "src_lengths": torch.tensor([200, 150], device=DEV)},
                  "target": torch.tensor([[5, 6, 7, 2], [8, 9, 2, 1]], device=DEV), "ntokens": 5}
        m.train()
        for it in range(2):  # the second step is counted (caches warm)
            m.flat.zero_grad()
            torch.cuda.synchronize()
            n0 = lib.launch_count()
            loss, _, _ = crit(m, sample)
            loss.backward()
            torch.cuda.synchronize()
            counts[rel] = lib.launch_count() - n0
    assert counts[True] - counts[False] == 8 * L, counts
