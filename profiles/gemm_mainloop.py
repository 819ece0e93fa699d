"""How fast does the GEMM mainloop run, against what cuBLAS reaches at the same shapes?

Records every ops.gemm call of one eager bench step (as profiles/gemm_epilogue_share.py does) and, for each distinct
configuration, times with CUDA events over graph-replayed back-to-back launches:

  t(K)      the call as recorded;
  main      t(2K) - t(K): the mainloop time of the call's K (operands re-allocated with twice the reduction extent);
  plain     the call at K with a plain bf16 store (no bias, activation, dropout, residual, skew or C2; accumulating
            calls keep their fp32 split-K accumulate);
  cuBLAS    torch.matmul on contiguous bf16 operands of the same batch x M x N x K, bf16 output;

and derives

  TFLOP/s   2 M N K nb / main (the mainloop rate) and 2 M N K nb / cuBLAS;
  clk/kb    clocks per k-block per CTA in the mainloop: main x (max SM clock) / (k-blocks of the call's K per CTA), with
            the tile width, multicast and K split the host picks (esp_gemm_bf16) and one CTA per SM.  The tensor cores
            need 2 x 128 x BN x 64 / 4096 clocks for a k-block (512 at BN = 128, 256 at BN = 64).

    python profiles/gemm_mainloop.py [--lib PATH] [--json OUT]

--lib times another build of the library (e.g. the parent commit's) for A/B runs.  GPU name, power limit and clocks are
read in the same run and printed first.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gemm_epilogue_share import make_variant, record_step_calls, time_us  # noqa: E402
from espresso_b200 import lib  # noqa: E402

BM, BK = 128, 64


def gpu_clocks():
    """name, power limit and SM clocks from nvidia-smi (max SM clock in MHz as a number, for the clock conversion)."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,clocks_throttle_reasons.active",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30, check=True)
    name, plim, cmax, csm, thr = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return dict(gpu=name, power_limit_w=float(plim), max_sm_clock_mhz=float(cmax), sm_clock_mhz=float(csm),
                throttle_reasons=thr)


def instance(M, N, K, nb, kw, sms):
    """(BN, MC, ksplit) as esp_gemm_bf16 picks them."""
    tm = -(-M // BM)
    tiles = lambda w: tm * -(-N // w) * nb  # noqa: E731
    num_kb = -(-K // BK)
    ksplit = 1
    if kw.get("accumulate"):
        bn = 128 if N > 64 else 64
        t = tiles(bn)
        best = -1.0
        ks = 1
        while ks <= max(num_kb // 4, 1) and (ks - 1) * t < sms:
            items = t * ks
            e = items / (-(-items // sms) * sms) - 0.01 * ks
            if e > best:
                best, ksplit = e, ks
            ks += 1
    elif N <= 64:
        bn = 64
    elif N <= 128 and tiles(128) * 10 < sms * 6 and tiles(64) < sms:
        bn = 64
    else:
        bn = 128
    bn = kw.get("tile_n") or bn
    mc = 2 if bn == 128 and (tm % 2 == 0 or tm >= 16) else 1
    return bn, mc, ksplit


def cublas_us(M, N, K, nb, launches, reps, dev):
    g = torch.Generator(device=dev).manual_seed(M + N + K)
    a = (torch.randn(nb, M, K, generator=g, device=dev) * 0.5).bfloat16()
    b = (torch.randn(nb, K, N, generator=g, device=dev) * 0.5).bfloat16()
    c = torch.empty(nb, M, N, device=dev, dtype=torch.bfloat16)
    return time_us(lambda: torch.matmul(a, b, out=c), launches, reps)


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
    info = gpu_clocks()
    info["lib"] = lib.LIB_PATH
    print(json.dumps(info))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    hz = info["max_sm_clock_mhz"] * 1e6
    calls = record_step_calls(dev)
    rows = []
    for i, (key, (cnt, call)) in enumerate(calls.items()):
        t = {}
        for which in "abc":
            gen = torch.Generator(device=dev).manual_seed(1000 + i)
            t[which] = time_us(make_variant(call, which, gen, dev), args.launches, args.reps)
        A, B, C_out, M, N, K, lda, ldb, ldc, kw = call
        nb = kw.get("nb1", 1) * kw.get("nb2", 1)
        t["cublas"] = cublas_us(M, N, K, nb, args.launches, args.reps, dev)
        torch.cuda.empty_cache()
        bn, mc, ks = instance(M, N, K, nb, kw, sms)
        items = -(-M // BM) * -(-N // bn) * nb * ks
        ctas = min(items, sms // mc * mc)
        kb_per_cta = items * (-(-K // BK) / ks) / ctas
        main = t["b"] - t["a"]
        flop = 2.0 * M * N * K * nb
        rows.append(dict(n=cnt, M=M, N=N, K=K, nb=nb, bn=bn, mc=mc, ksplit=ks,
                         epi=" ".join(k for k in ("bias", "C2", "aux", "R", "rowsum_a") if kw.get(k) is not None)
                         + (" act%d" % kw["act"] if kw.get("act") else "") + (" drop" if kw.get("drop_p", 0) > 0 else "")
                         + (" acc" if kw.get("accumulate") else "") + (" f32" if C_out.dtype == torch.float32 else ""),
                         us_k=t["a"], us_2k=t["b"], main=main, plain=t["c"], cublas=t["cublas"],
                         main_tflops=flop / main / 1e6 if main > 0 else float("nan"), cublas_tflops=flop / t["cublas"] / 1e6,
                         clk_per_kb=main * 1e-6 * hz / kb_per_cta if main > 0 else float("nan"),
                         ideal_clk_per_kb=2 * BM * bn * BK / 4096))
    rows.sort(key=lambda r: -r["n"] * r["us_k"])
    print("| n | M × N × K | nb | BN MC ks | epilogue | t(K) µs | mainloop µs | plain µs | cuBLAS µs | mainloop TFLOP/s "
          "| cuBLAS TFLOP/s | clk/kb (ideal) |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %d | %d × %d × %d | %d | %d %d %d | %s | %.1f | %.1f | %.1f | %.1f | %.0f | %.0f | %.0f (%d) |"
              % (r["n"], r["M"], r["N"], r["K"], r["nb"], r["bn"], r["mc"], r["ksplit"], r["epi"].strip(), r["us_k"],
                 r["main"], r["plain"], r["cublas"], r["main_tflops"], r["cublas_tflops"], r["clk_per_kb"],
                 r["ideal_clk_per_kb"]))
    tot = {k: sum(r["n"] * r[k] for r in rows) / 1e3 for k in ("us_k", "main", "plain", "cublas")}
    summary = {"launches": sum(r["n"] for r in rows), "configs": len(rows), "gemm_ms": tot["us_k"],
               "mainloop_ms": tot["main"], "plain_ms": tot["plain"], "cublas_ms": tot["cublas"]}
    print(json.dumps({"per_step": {k: (round(v, 3) if isinstance(v, float) else v) for k, v in summary.items()}}))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"info": info, "rows": rows, "per_step": summary}, f, indent=1)


if __name__ == "__main__":
    main()
