"""Do two builds of the library compute the same GEMMs?  Replays every distinct ops.gemm configuration of one eager bench
step (recorded as profiles/gemm_epilogue_share.py records them) through the in-tree library and through --other-lib, on
the same seeded operands, and compares the outputs: C and C2 of every non-accumulating call bit for bit; the split-K
fp32 outputs and bias-gradient row sums (their `red` order varies between runs) to 1e-5 of their largest magnitude.

    python profiles/gemm_ab_bitexact.py --other-lib PATH

PATH is another build of libespresso_b200.so, e.g. the parent commit's: `git worktree add /tmp/parent HEAD~1 &&
make -C /tmp/parent/espresso_b200/csrc`.  Exits non-zero on any difference.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gemm_epilogue_share import TENSOR_KW, record_step_calls, seeded_like  # noqa: E402
from espresso_b200 import lib, ops  # noqa: E402


def run(handle, call, seed, dev):
    """Outputs of one call through library `handle` on operands and output buffers seeded by `seed`."""
    A, B, C_out, M, N, K, lda, ldb, ldc, kw = call
    gen = torch.Generator(device=dev).manual_seed(seed)
    kw = dict(kw)
    for k in TENSOR_KW:
        if kw.get(k) is not None:
            kw[k] = seeded_like(kw[k], gen)
    A, B, C = seeded_like(A, gen), seeded_like(B, gen), seeded_like(C_out, gen)
    saved = lib._lib
    lib._lib = handle
    try:
        ops.gemm(A, B, C, M, N, K, lda, ldb, ldc, **kw)
    finally:
        lib._lib = saved
    torch.cuda.synchronize()
    return {"C": C, "C2": kw.get("C2"), "rowsum_a": kw.get("rowsum_a")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other-lib", required=True)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    calls = record_step_calls(dev)
    mine = lib.load()
    lib._lib, lib.LIB_PATH = None, os.path.abspath(args.other_lib)
    other = lib.load()
    lib._lib = mine
    n_exact = n_tol = 0
    worst_tol = 0.0
    bad = []
    for i, (key, (cnt, call)) in enumerate(calls.items()):
        x, y = run(mine, call, 5000 + i, dev), run(other, call, 5000 + i, dev)
        acc = call[9].get("accumulate", False)
        for name in ("C", "C2", "rowsum_a"):
            if x[name] is None:
                continue
            if acc:
                scale = float(y[name].abs().max()) or 1.0
                d = float((x[name] - y[name]).abs().max()) / scale
                worst_tol = max(worst_tol, d)
                n_tol += 1
                if d > 1e-5:
                    bad.append((key[:3], name, d))
            else:
                n_exact += 1
                if not torch.equal(x[name], y[name]):
                    bad.append((key[:3], name, float((x[name].float() - y[name].float()).abs().max())))
    print(json.dumps({"configs": len(calls), "launches": sum(c for c, _ in calls.values()),
                      "outputs_compared_exactly": n_exact, "accumulating_outputs": n_tol, "n_differences": len(bad),
                      "accumulating_max_rel_diff": worst_tol, "differences": bad[:20]}))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
