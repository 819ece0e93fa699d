"""Attention without positions (absolute-position encoders) against the relative-position kernels, on the H100.

    python profiles/abspos_attn_bench.py [--reps N] [--steps N] [--out FILE]

1. Per-launch device time (CUDA events over back-to-back launches) of the fused attention forward and of its score-side
   backward without positions (esp_attn_fused_fwd with pos == NULL, esp_attn_fused_bwd with dbd == NULL) against the
   relative-position kernels given an all-zero position table, at WSJ-like (d = 256, 4 heads) and LibriSpeech-like
   (d = 512, 8 heads) batch shapes.  The two arms alternate inside one run, several rounds each; the median is reported.
2. Milliseconds per training step of a WSJ-shaped model (Transformer 12 x 256 encoder with absolute positions, 6-layer
   decoder with relaxed encoder attention 0.35, temporal label smoothing), eager and replayed from a CUDA graph.

Records the card's name and power limit with the numbers; prints one JSON object (and writes it to --out if given)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from espresso_b200 import ops  # noqa: E402

DEV = torch.device("cuda:0")
# (label, B, T', H): WSJ-like (d 256 / 4 heads, utterances up to ~16 s -> T' ~ 400) and the LibriSpeech bench's shapes
SHAPES = [("wsj_32x200", 32, 200, 4), ("wsj_16x400", 16, 400, 4), ("libri_15x431", 15, 431, 8), ("libri_8x754", 8, 754, 8)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": out}


def time_launches(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / reps  # us per launch


def kernels(reps, rounds):
    res = {}
    for label, B, T, H in SHAPES:
        d = H * 64
        g = torch.Generator(device="cpu").manual_seed(T)
        qkv = (torch.randn(B * T, 3 * d, generator=g) * 0.7).bfloat16().to(DEV)
        qu = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16().to(DEV)
        dctx = (torch.randn(B * T, d, generator=g) * 0.5).bfloat16().to(DEV)
        lens = torch.randint(T // 2, T + 1, (B,), generator=g, dtype=torch.int32)
        lens[0] = T
        lens = lens.to(DEV)
        k, v = qkv[:, d:2 * d], qkv[:, 2 * d:]
        zeros = torch.zeros(2 * T - 1, 64, dtype=torch.bfloat16, device=DEV)
        ldp = (2 * T - 1 + 7) // 8 * 8
        drop = 0.1
        ctx, p, pd = ops.attn_fused_fwd(qu, None, k, v, None, B, T, H, lens, drop_p=drop, seed=1)
        ctx_r, p_r, pd_r = ops.attn_fused_fwd(qu, qu, k, v, zeros, B, T, H, lens, drop_p=drop, seed=1, pos_hstride=0)
        assert torch.equal(ctx, ctx_r) and torch.equal(p, p_r) and torch.equal(pd, pd_r)
        dqkv = torch.empty(B * T, 3 * d, dtype=torch.bfloat16, device=DEV)
        arms = {
            "fwd_nopos": lambda: ops.attn_fused_fwd(qu, None, k, v, None, B, T, H, lens, drop_p=drop, seed=1),
            "fwd_relpos_zero_table": lambda: ops.attn_fused_fwd(qu, qu, k, v, zeros, B, T, H, lens, drop_p=drop, seed=1,
                                                                pos_hstride=0),
            # the backward entry: row dots + the fused kernel (+ the skew copy of dS for relative positions)
            "bwd_nopos": lambda: ops.attn_fused_bwd(dctx, ctx, qu, v, p, pd, B, T, H, None, dqkv[:, d:2 * d], dqkv[:, 2 * d:],
                                                    drop_p=drop, seed=1),
            "bwd_relpos": lambda: ops.attn_fused_bwd(dctx, ctx, qu, v, p, pd, B, T, H, ldp, dqkv[:, d:2 * d], dqkv[:, 2 * d:],
                                                     drop_p=drop, seed=1),
        }
        samples = {n: [] for n in arms}
        for _ in range(rounds):  # alternate the arms
            for n, fn in arms.items():
                samples[n].append(time_launches(fn, reps))
        r = {n: {"us_median": float(np.median(s)), "us_min": float(np.min(s)), "us_max": float(np.max(s))}
             for n, s in samples.items()}
        r["fwd_speedup"] = r["fwd_relpos_zero_table"]["us_median"] / r["fwd_nopos"]["us_median"]
        r["bwd_speedup"] = r["bwd_relpos"]["us_median"] / r["bwd_nopos"]["us_median"]
        r["shape"] = {"B": B, "T": T, "H": H, "head_dim": 64, "attention_dropout": drop}
        res[label] = r
    return res


def wsj_step(steps):
    """ms per training step of a WSJ-shaped model, eager and CUDA-graphed (same batch)."""
    from espresso_b200.criterions import LabelSmoothedCrossEntropyV2Criterion
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerModelBase
    from espresso_b200.optim import NoamLRScheduler
    from espresso_b200.trainer import Trainer

    V = 52

    class _Dict:
        def __len__(self):
            return V

        def pad(self):
            return 1

        def eos(self):
            return 2

        def unk(self):
            return 3

    class _Task:
        feat_dim, feat_in_channels, target_dictionary = 80, 1, _Dict()

    cfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.2, attention_dropout=0.0, activation_dropout=0.0, max_source_positions=3600, max_target_positions=1024,
        encoder=dict(embed_dim=256, ffn_embed_dim=1024, layers=12, attention_heads=4, normalize_before=True,
                     relative_positional_embeddings=False, layer_type="transformer"),
        decoder=dict(embed_dim=256, ffn_embed_dim=1024, layers=6, attention_heads=4, normalize_before=True,
                     input_dim=256, output_dim=256, relaxed_attention_weight=0.35)))
    torch.manual_seed(0)
    m = SpeechTransformerModelBase.build_model(cfg, _Task()).finalize_(DEV)
    crit = LabelSmoothedCrossEntropyV2Criterion(_Task(), label_smoothing=0.05, smoothing_type="temporal")
    rs = np.random.RandomState(0)
    B, T, U = 24, 1200, 96  # ~12 s utterances (T' = 300 after 4x subsampling), 96 characters
    lens = torch.from_numpy(rs.randint(T // 2, T + 1, size=B)).sort(descending=True).values
    lens[0] = T
    tgt = torch.full((B, U), 1, dtype=torch.long)
    prev = torch.full((B, U), 1, dtype=torch.long)
    for b in range(B):
        u = int(rs.randint(U // 2, U))
        toks = torch.from_numpy(rs.randint(4, V, size=u))
        tgt[b, :u], tgt[b, u] = toks, 2
        prev[b, 0], prev[b, 1:u + 1] = 2, toks
    sample = {"net_input": {"src_tokens": torch.from_numpy(rs.randn(B, T, 80).astype(np.float32)).to(DEV),
                            "src_lengths": lens.to(DEV), "src_lengths_cpu": lens, "prev_output_tokens": prev.to(DEV),
                            "prev_output_tokens_cpu": prev},
              "target": tgt.to(DEV)}
    out = {"shape": {"B": B, "frames": T, "tokens": U, "encoder": "12 x 256 (4 heads, abs. positions)",
                     "decoder": "6 x 256, relaxed encoder attention 0.35"}}
    for mode in ("eager", "graphed"):
        tr = Trainer(m, crit, NoamLRScheduler(5.0, 25000, 256, 1e-6), use_cuda_graphs=(mode == "graphed"),
                     bucket_frames=T, bucket_tokens=U)
        for _ in range(3):
            tr.train_step([sample])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            tr.train_step([sample])
        torch.cuda.synchronize()
        out[mode + "_ms_per_step"] = (time.perf_counter() - t0) * 1e3 / steps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    res = {"card": card(), "kernels_us_per_launch": kernels(a.reps, a.rounds), "wsj_step": wsj_step(a.steps)}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
