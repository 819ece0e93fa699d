"""Where do the GEMM's MMA and epilogue warpgroups spend their clocks?  Per-role phase clocks of a profiling build of
csrc/gemm_tcgen05.cu (-DESP_GEMM_PHASES), at the non-accumulating configurations of one eager bench step with
K = 512 or 2048 (recorded as profiles/gemm_epilogue_share.py records them).

    python profiles/gemm_phases.py [--lib PATH] [--launches N] [--json OUT]

Without --lib the script compiles gemm_tcgen05.cu with the flag into a temporary directory and links it with the other
objects of the in-tree build (espresso_b200/csrc/build, made by build()); --lib runs another profiling build instead.
Thread 0 of each MMA warpgroup and of each epilogue warpgroup counts, per CTA:

  acc wait    clocks the MMA warpgroup waits on acc_empty before it stages a finished tile, as a share of its work loop;
  epi busy    clocks the epilogue warpgroup spends on a tile (or tile half) it serves: from acc_full to its acc_empty
              arrive, per tile served and as a share of its work loop.

The clock reads cost a little themselves, so the launch times of that build are not the kernel's."""
import argparse
import ctypes
import json
import os
import shutil
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gemm_epilogue_share import make_variant, record_step_calls  # noqa: E402
from espresso_b200 import lib  # noqa: E402

PHASES = ["mma_acc_wait", "mma_loop", "epi_busy", "epi_loop", "epi_tiles"]


def build_phase_lib(out_dir):
    """gemm_tcgen05.cu with the phase clocks, linked with the in-tree build's other objects (same flags as csrc/Makefile)."""
    csrc = os.path.join(ROOT, "espresso_b200", "csrc")
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    arch = ["-gencode", "arch=compute_90a,code=sm_90a"]
    obj = os.path.join(out_dir, "gemm_tcgen05.o")
    subprocess.check_call([nvcc] + arch + ["-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-I" + os.path.join(ROOT, "include"),
                                           "-I" + csrc, "--expt-relaxed-constexpr", "-DESP_GEMM_PHASES", "-c",
                                           os.path.join(csrc, "gemm_tcgen05.cu"), "-o", obj])
    others = sorted(os.path.join(csrc, "build", f) for f in os.listdir(os.path.join(csrc, "build"))
                    if f.endswith(".o") and f != "gemm_tcgen05.o")
    lib_path = os.path.join(out_dir, "libespresso_b200.so")
    subprocess.check_call([nvcc] + arch + ["-shared", "-o", lib_path, obj] + others + ["-lcudart"])
    return lib_path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="a profiling build to run instead of building one")
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the rows as JSON here")
    args = ap.parse_args()
    if args.lib:
        lib.LIB_PATH = os.path.abspath(args.lib)
        lib.load()
    else:
        tmp = tempfile.mkdtemp(prefix="gemm_phases_")
        try:
            lib.LIB_PATH = build_phase_lib(tmp)
            lib.load()
        finally:
            shutil.rmtree(tmp, ignore_errors=True)
    buf = (ctypes.c_ulonglong * len(PHASES))()

    def phase_clk():
        lib.check(lib.load().esp_gemm_phase_clk(buf))
        return dict(zip(PHASES, (int(v) for v in buf)))

    dev = torch.device("cuda:0")
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev), "lib": lib.LIB_PATH}))
    calls = record_step_calls(dev)
    rows = []
    for i, (key, (cnt, call)) in enumerate(calls.items()):
        A, B, C_out, M, N, K, lda, ldb, ldc, kw = call
        if kw.get("accumulate") or K not in (512, 2048) or kw.get("nb1", 1) * kw.get("nb2", 1) != 1:
            continue
        fn = make_variant(call, "a", torch.Generator(device=dev).manual_seed(1000 + i), dev)
        fn()
        torch.cuda.synchronize()
        phase_clk()  # reset
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        c = phase_clk()
        rows.append(dict(n=cnt, M=M, N=N, K=K,
                         epi=(" ".join(k for k in ("bias", "C2", "aux", "R") if kw.get(k) is not None)
                              + (" act%d" % kw["act"] if kw.get("act") else "")
                              + (" drop" if kw.get("drop_p", 0) > 0 else "")).strip(),
                         us_profiling_build=e0.elapsed_time(e1) * 1e3 / args.launches,
                         mma_acc_wait_share=c["mma_acc_wait"] / max(c["mma_loop"], 1),
                         epi_busy_share=c["epi_busy"] / max(c["epi_loop"], 1),
                         epi_kclk_per_tile=c["epi_busy"] / max(c["epi_tiles"], 1) / 1e3, clk=c))
        torch.cuda.empty_cache()
    rows.sort(key=lambda r: (r["K"], -r["n"] * r["us_profiling_build"]))
    print("| n | M × N × K | epilogue | µs (profiling build) | MMA acc_empty wait | epilogue busy | epilogue kclk per tile served |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %d | %d × %d × %d | %s | %.1f | %.0f %% | %.0f %% | %.1f |"
              % (r["n"], r["M"], r["N"], r["K"], r["epi"] or "none", r["us_profiling_build"],
                 100 * r["mma_acc_wait_share"], 100 * r["epi_busy_share"], r["epi_kclk_per_tile"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
