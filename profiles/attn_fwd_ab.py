"""Fused rel-pos attention forward (csrc/attn_fused.cu) at the bench's batch shapes: device time per launch (CUDA events
over back-to-back launches), useful TFLOP/s and the ratio of the MMA work the kernel executes to the useful work.

    python profiles/attn_fwd_ab.py [--reps N] [--phases]

Useful flops per (utterance, head) are 2 hd (T'^2 + T'(2T'-1) + T'^2), as bench.useful_gemm_flops counts them: Qu K^T,
Qv Pos^T over the 2T'-1 relative positions, P V.  "executed_w_once" is what the wgmma instructions of the current kernel
compute: per CTA (128 query rows) and pass, one 128 x 128 x 64 W half per key tile plus one extra half at the pass start,
S per key tile, and P V per key tile in pass 2; tiles are full even where T' is ragged.  (The kernel before its Hopper
rework computed two W halves per key tile: run against that library, these two columns do not describe it.)

--phases compiles a profiling build of the library (-DESP_ATTN_FWD_PHASES) into a temporary directory and prints, per
shape, the share of the math warpgroups' SM clocks spent in each phase of the key-tile loop and the clocks per CTA.  The
clock reads and their bookkeeping cost time themselves (that build spills a little), so the shares are indicative and
the launch times of that build are not the kernel's."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from espresso_b200 import ops  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = [(15, 431), (24, 250), (8, 754)]
PHASES = ["W (TMA wait + MMA)", "W stage (bf16 stores)", "S (TMA wait + MMA)", "logits (skew, mask)",
          "pass-1 max / sum", "pass-2 P, dropout, P/Pd stores", "P V issue (V wait)", "W move"]


def build_phase_lib(out_dir):
    """The whole library with the fused forward's phase clocks compiled in (same flags as csrc/Makefile)."""
    csrc = os.path.join(ROOT, "espresso_b200", "csrc")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"]
    flags = arch + ["-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-I" + os.path.join(ROOT, "include"), "-I" + csrc,
                    "--expt-relaxed-constexpr", "-DESP_ATTN_FWD_PHASES"]
    srcs = sorted(f for f in os.listdir(csrc) if f.endswith(".cu"))
    objs = [os.path.join(out_dir, f[:-3] + ".o") for f in srcs]
    with ThreadPoolExecutor(max_workers=4) as ex:
        list(ex.map(lambda so: subprocess.check_call([nvcc] + flags + ["-c", os.path.join(csrc, so[0]), "-o", so[1]]),
                    zip(srcs, objs)))
    lib_path = os.path.join(out_dir, "libespresso_b200.so")
    subprocess.check_call([nvcc] + arch + ["-shared", "-o", lib_path] + objs + ["-lcudart"])
    return lib_path


H, HD = 8, 64


def flops(B, T):
    nkt = (T + 127) // 128
    useful = 2.0 * B * H * HD * (T * T + T * (2 * T - 1) + T * T)
    tile = 2.0 * 128 * 128 * HD
    executed = B * H * nkt * tile * (2 * (nkt + 1) + 2 * nkt + nkt)
    return useful, executed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--phases", action="store_true", help="per-phase clock shares from a profiling build")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    phase_clk = None
    if args.phases:
        import ctypes

        from espresso_b200 import lib

        tmp = tempfile.mkdtemp(prefix="attn_fwd_phases_")
        try:
            lib.LIB_PATH = build_phase_lib(tmp)
            lib.load()
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
        buf = (ctypes.c_ulonglong * len(PHASES))()

        def phase_clk():
            lib.check(lib.load().esp_attn_fwd_phase_clk(buf))
            return [int(v) for v in buf]
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev)}))
    d = H * HD
    for B, T in SHAPES:
        g = torch.Generator(device="cpu").manual_seed(T)
        qkv = (torch.randn(B * T, 3 * d, generator=g) * 0.7).bfloat16().to(dev)
        qu = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16().to(dev)
        qv = (torch.randn(B * T, d, generator=g) * 0.3).bfloat16().to(dev)
        pos = (torch.randn(2 * T - 1, d, generator=g) * 0.7).bfloat16().to(dev)
        lens = torch.randint(T // 2, T + 1, (B,), generator=g, dtype=torch.int32)
        lens[0] = T
        lens = lens.to(dev)
        useful, executed = flops(B, T)
        for drop in (0.0, 0.1):
            fn = lambda: ops.attn_fused_fwd(qu, qv, qkv[:, d:2 * d], qkv[:, 2 * d:], pos, B, T, H, lens,  # noqa: E731
                                            drop_p=drop, seed=11)
            for _ in range(5):
                fn()
            torch.cuda.synchronize()
            if phase_clk:
                phase_clk()  # reset
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(int(1e8))  # the host runs ahead: back-to-back launches, no launch gaps in the window
            e0.record()
            for _ in range(args.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / args.reps
            res = {"B": B, "T": T, "dropout": drop, "us_per_launch": round(us, 1),
                   "useful_tflops": round(useful / us / 1e6, 1), "executed_w_once_tflops": round(executed / us / 1e6, 1),
                   "executed_w_once_over_useful": round(executed / useful, 3)}
            if phase_clk:
                clk = phase_clk()
                ctas = (T + 127) // 128 * H * B * args.reps
                res["phase_share"] = {n: round(c / sum(clk), 3) for n, c in zip(PHASES, clk)}
                res["kclk_per_cta"] = round(sum(clk) / (2 * ctas) / 1e3, 1)  # two math warpgroups per CTA
                res["us_per_launch_of_profiling_build"] = res.pop("us_per_launch")
            print(json.dumps(res))


if __name__ == "__main__":
    main()
