"""How much of the bench step's GEMM time is per-tile fixed cost (fused epilogue + pipeline fill) that overlapping the
epilogue with the next tile's MMAs could recover?

Records every ops.gemm call of one eager step of the bench workload (the first bench batch), then, for each distinct
configuration, allocates its own seeded operands and times three variants with CUDA events over back-to-back launches
(a CUDA graph of --launches launches, warmed, replayed --reps times):

  (a) the call as recorded, at its reduction length K;
  (b) the same call at 2K (A and B re-allocated with twice the reduction extent, same majors and batch broadcasting);
  (c) the call at K with a plain bf16 store: no bias, activation, dropout, residual, skew or C2.  An accumulating
      (split-K, fp32 `red`) call keeps its fp32 accumulate, which decides its K split, and drops only the row sums.

and prints per configuration and summed over the step (count x time):

  mainloop           t(2K) - t(K)
  fixed per tile     2 t(K) - t(2K)   epilogue + pipeline fill + wave tail: what overlap can recover at most
  epilogue extra     t(a) - t(c)      the fused epilogue's cost over a plain store

    python profiles/gemm_epilogue_share.py [--lib PATH] [--json OUT]

--lib times another build of the library (e.g. the parent commit's, built with `make -C <worktree>/espresso_b200/csrc`).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from espresso_b200 import lib, ops  # noqa: E402

TENSOR_KW = ("bias", "aux", "R", "C2", "rowsum_a")


def _tdesc(t):
    return None if t is None else (str(t.dtype), tuple(t.shape), tuple(t.stride()), t.storage_offset() % 64)


def call_key(M, N, K, lda, ldb, ldc, C_out, kw):
    """Everything that determines what a call computes and how, except where its tensors live."""
    items = []
    for k in sorted(kw):
        v = kw[k]
        items.append((k, _tdesc(v) if torch.is_tensor(v) or k in TENSOR_KW else v))
    return (M, N, K, lda, ldb, ldc, str(C_out.dtype), tuple(items))


def record_step_calls(dev):
    """{key: [count, (A, B, C_out, M, N, K, lda, ldb, ldc, kw)]} of every ops.gemm call of one eager bench step."""
    from espresso_b200.criterions import CtcLossCriterion
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel
    from espresso_b200.optim import NoamLRScheduler
    from espresso_b200.trainer import Trainer

    lib.load()
    torch.manual_seed(1)
    cfg = SpeechTransformerConfig.from_dict(dict(dropout=0.1, attention_dropout=0.1, activation_dropout=0.1,
                                                 layernorm_embedding=True, encoder=dict(bench.MODEL)))
    model = SpeechTransformerEncoderModel.build_model(cfg, bench._Task()).finalize_(dev)
    model.frontend = OnTheFlyFbank(np.full(80, 15.0), np.full(80, 4.0))
    trainer = Trainer(model, CtcLossCriterion(bench._Task()), NoamLRScheduler(5.0, 25000, 512, 1e-6),
                      adam_betas=(0.9, 0.98), clip_norm=2.0, use_cuda_graphs=False)
    b = bench.make_batches(1)[0]
    d = {k: (torch.from_numpy(v).to(dev) if isinstance(v, np.ndarray) else v) for k, v in b.items()}
    sample = {"net_input": {"src_tokens": d["wave"], "src_lengths": d["n_samples"], "freq_masks": d["fm"],
                            "time_masks": d["tm"], "src_lengths_cpu": torch.from_numpy(b["n_samples"]).long()},
              "target": d["target"]}
    trainer.train_step([sample])  # warm
    calls = {}
    real = ops.gemm

    def rec(A, B, C_out, M, N, K, lda, ldb, ldc, **kw):
        key = call_key(M, N, K, lda, ldb, ldc, C_out, kw)
        if key not in calls:
            calls[key] = [0, (A, B, C_out, M, N, K, lda, ldb, ldc, dict(kw))]
        calls[key][0] += 1
        return real(A, B, C_out, M, N, K, lda, ldb, ldc, **kw)

    ops.gemm = rec
    try:
        trainer.train_step([sample])
    finally:
        ops.gemm = real
    torch.cuda.synchronize()
    return calls


def seeded_like(t, gen, scale=0.5, dtype=None):
    """A fresh tensor with t's shape and strides (and its alignment within the storage) over seeded values."""
    off = t.storage_offset() % 64
    n = off + 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride()))
    flat = (torch.randn(n, generator=gen, device=t.device) * scale).to(dtype or t.dtype)
    return torch.as_strided(flat, t.shape, t.stride(), off)


def operand_2k(kmajor, rows_k, rows_mn, ld, nb1, nb2, s, gen, dev, k):
    """Dense seeded operand of reduction length k (K-major: rows_mn rows of k; MN-major: k rows of rows_mn), with the
    recorded call's batch broadcasting; returns (tensor, ld, (s1, s2))."""
    if kmajor:
        ld2 = max(ld, -(-k // 8) * 8)
        per = rows_mn * ld2
    else:
        ld2 = ld
        per = k * ld2
    b1, b2 = (nb1 > 1 and s[0] != 0), (nb2 > 1 and s[1] != 0)
    s1 = per if b1 else 0
    s2 = per * (nb1 if b1 else 1) if b2 else 0
    total = per * (nb1 if b1 else 1) * (nb2 if b2 else 1)
    t = (torch.randn(total, generator=gen, device=dev) * 0.5).bfloat16()
    return t, ld2, (s1, s2)


def make_variant(call, which, gen, dev):
    """Zero-argument launcher of variant `which` ('a', 'b', 'c') of a recorded call on freshly seeded operands."""
    A, B, C_out, M, N, K, lda, ldb, ldc, kw = call
    kw = dict(kw)
    for k in TENSOR_KW:
        if kw.get(k) is not None:
            kw[k] = seeded_like(kw[k], gen) if k != "rowsum_a" else torch.zeros_like(kw[k])
    C = seeded_like(C_out, gen)
    nb1, nb2 = kw.get("nb1", 1), kw.get("nb2", 1)
    ak, bk = kw.get("a_kmajor", True), kw.get("b_kmajor", True)
    if which == "b":
        A2, lda2, sA = operand_2k(ak, 2 * K, M, lda, nb1, nb2, kw.get("sA", (0, 0)), gen, dev, 2 * K)
        B2, ldb2, sB = operand_2k(bk, 2 * K, N, ldb, nb1, nb2, kw.get("sB", (0, 0)), gen, dev, 2 * K)
        kw["sA"], kw["sB"] = sA, sB
        args = (A2, B2, C, M, N, 2 * K, lda2, ldb2, ldc)
    else:
        args = (seeded_like(A, gen), seeded_like(B, gen), C, M, N, K, lda, ldb, ldc)
    if which == "c":
        for k in ("bias", "aux", "R", "C2", "rowsum_a"):
            kw.pop(k, None)
        for k in ("sAux", "sR", "ld_aux", "ldr", "skew_r", "drop_p", "drop_mode", "alpha", "beta", "act"):
            kw.pop(k, None)
        if not kw.get("accumulate", False) and C.dtype != torch.bfloat16:
            args = args[:2] + (seeded_like(C, gen, dtype=torch.bfloat16),) + args[3:]
    return lambda: ops.gemm(*args, **kw)


def time_us(fn, launches, reps):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(launches):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (launches * reps)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:  # the table is still worth printing
        q = "nvidia-smi unavailable: %r" % ex
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="library to time instead of the in-tree build")
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the rows as JSON here")
    args = ap.parse_args()
    if args.lib:
        lib.LIB_PATH = os.path.abspath(args.lib)
    dev = torch.device("cuda:0")
    calls = record_step_calls(dev)
    info = {"gpu": gpu_info(), "lib": lib.LIB_PATH}
    print(json.dumps(info))
    rows = []
    for i, (key, (cnt, call)) in enumerate(calls.items()):
        t = {}
        for which in "abc":
            gen = torch.Generator(device=dev).manual_seed(1000 + i)
            t[which] = time_us(make_variant(call, which, gen, dev), args.launches, args.reps)
        torch.cuda.empty_cache()
        A, B, C_out, M, N, K, lda, ldb, ldc, kw = call
        rows.append(dict(n=cnt, M=M, N=N, K=K, nb=kw.get("nb1", 1) * kw.get("nb2", 1),
                         ak=int(kw.get("a_kmajor", True)), bk=int(kw.get("b_kmajor", True)),
                         epi=" ".join(k for k in ("bias", "C2", "aux", "R", "rowsum_a") if kw.get(k) is not None)
                         + (" act%d" % kw["act"] if kw.get("act") else "") + (" drop" if kw.get("drop_p", 0) > 0 else "")
                         + (" acc" if kw.get("accumulate") else "") + (" f32" if C_out.dtype == torch.float32 else ""),
                         us_a=t["a"], us_2k=t["b"], us_c=t["c"], main=t["b"] - t["a"], fixed=2 * t["a"] - t["b"],
                         epi_extra=t["a"] - t["c"]))
    rows.sort(key=lambda r: -r["n"] * r["us_a"])
    print("| n | M | N | K | nb | aK bK | epilogue | t(K) us | t(2K) us | plain us | mainloop us | fixed us | epi extra us |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %d | %d | %d | %d | %d | %d %d | %s | %.1f | %.1f | %.1f | %.1f | %.1f | %.1f |"
              % (r["n"], r["M"], r["N"], r["K"], r["nb"], r["ak"], r["bk"], r["epi"].strip(), r["us_a"], r["us_2k"],
                 r["us_c"], r["main"], r["fixed"], r["epi_extra"]))
    tot = {k: sum(r["n"] * r[k] for r in rows) / 1e3 for k in ("us_a", "main", "fixed", "epi_extra")}
    k512 = {k: sum(r["n"] * r[k] for r in rows if r["K"] == 512 and "acc" not in r["epi"]) / 1e3
            for k in ("us_a", "main", "fixed", "epi_extra")}
    summary = {"launches": sum(r["n"] for r in rows), "configs": len(rows), "gemm_ms": tot["us_a"],
               "mainloop_ms": tot["main"], "fixed_ms": tot["fixed"], "epi_extra_ms": tot["epi_extra"],
               "k512_gemm_ms": k512["us_a"], "k512_fixed_ms": k512["fixed"], "k512_epi_extra_ms": k512["epi_extra"]}
    print(json.dumps({"per_step": {k: (round(v, 3) if isinstance(v, float) else v) for k, v in summary.items()}}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"info": info, "rows": rows, "per_step": summary}, f, indent=1)


if __name__ == "__main__":
    main()
