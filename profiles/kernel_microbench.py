"""Device-time microbenchmark of the non-GEMM kernels at the bench workload's shapes.

Each op is captured NREP times in one CUDA graph over rotating input sets (larger than the 126 MB L2 together), the
graph is replayed and timed with CUDA events: no host launch gaps, no profiler serialisation.  Prints us per launch
and the algorithmic GB/s (bytes the op must read + write once).

    python profiles/kernel_microbench.py            # on the GPU
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from espresso_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
B, T, D, H, FF, KS = 24, 272, 512, 8, 2048, 31
R = B * T
NREP = 24


def bf(*shape):
    return torch.randn(*shape, device=dev, dtype=torch.bfloat16)


ONCE = os.environ.get("KMB_ONCE") == "1"  # two plain launches per op and no timing: the mode to run under ncu


def timed(name, make_inputs, fn, nbytes, nsets=8):
    if ONCE:
        args = make_inputs()
        fn(*args)
        fn(*args)
        torch.cuda.synchronize()
        return
    sets = [make_inputs() for _ in range(nsets)]
    for i in range(2):
        fn(*sets[i % nsets])
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for i in range(NREP):
            fn(*sets[i % nsets])
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (5 * NREP)
    print("%-34s %8.2f us   %7.0f GB/s   (%.1f MB)" % (name, us, nbytes / us / 1e3, nbytes / 1e6))


lens = torch.full((B,), T, device=dev, dtype=torch.int32)
gamma, beta = bf(D), bf(D)
acc = [torch.zeros(4096, device=dev, dtype=torch.float32) for _ in range(2)]

for N in (512, 1536, 2048):
    timed("colsum [R,%d]" % N, lambda N=N: (bf(R, N),), lambda x: ops.colsum(x, acc[0][: x.shape[1]]), R * N * 2)
timed("layer_norm_fwd", lambda: (bf(R, D),), lambda x: ops.layer_norm_fwd(x, gamma, beta), R * D * 4)
timed("layer_norm_fwd +mask+dropout", lambda: (bf(R, D),),
      lambda x: ops.layer_norm_fwd(x, gamma, beta, lens=lens, T=T, drop_p=0.1, seed=3), R * D * 4)


def ln_in():
    x = bf(R, D)
    _, m, r = ops.layer_norm_fwd(x, gamma, beta)
    return bf(R, D), x, m, r, bf(R, D)


timed("layer_norm_bwd (+dres)", ln_in,
      lambda dy, x, m, r, dres: ops.layer_norm_bwd(dy, x, m, r, gamma, acc[0][:D], acc[1][:D], dres=dres), R * D * 8)
timed("dropout [R,512]", lambda: (bf(R, D),), lambda x: ops.dropout(x, 0.1, 5), R * D * 4)
timed("dropout [R,2048]", lambda: (bf(R, FF),), lambda x: ops.dropout(x, 0.1, 5), R * FF * 4)

ld = (T + 7) // 8 * 8
timed("attn_softmax_fwd (dropout)", lambda: (bf(H, B, T, ld),),
      lambda s: ops.attn_softmax_fwd(s, T, lens, drop_p=0.1, seed=7), H * B * T * ld * 6, nsets=6)
ldp = (2 * T - 1 + 7) // 8 * 8
timed("attn_softmax_bwd (+dBD)", lambda: (torch.softmax(bf(H, B, T, ld).float(), -1).bfloat16(), bf(H, B, T, ld)),
      lambda p, dp: ops.attn_softmax_bwd(p, dp, T, ldp, drop_p=0.1, seed=7),
      H * B * T * ld * 6 + H * B * T * ldp * 2, nsets=6)

w = bf(D, KS)
dwacc = torch.zeros(D, KS, device=dev, dtype=torch.float32)
timed("glu_dwconv_fwd", lambda: (bf(B, T, 2 * D),), lambda g: ops.glu_dwconv_fwd(g, w), R * D * 6)
timed("glu_dwconv_bwd", lambda: (bf(B, T, D), bf(B, T, 2 * D)), lambda dy, g: ops.glu_dwconv_bwd(dy, g, w, dwacc),
      R * D * 10)
mr = torch.stack([torch.zeros(D, device=dev), torch.ones(D, device=dev)]).contiguous()
timed("bn_act_fwd (SiLU)", lambda: (bf(B, T, D),), lambda y: ops.bn_act_fwd(y, mr, gamma, beta), R * D * 4)
timed("bn_act_bwd (reduce+apply)", lambda: (bf(B, T, D), bf(B, T, D)),
      lambda dz, y: ops.bn_act_bwd(dz, y, mr, gamma, beta, acc[0][:D], acc[1][:D]), R * D * 10)
u, v = bf(D), bf(D)
timed("qprep_fwd", lambda: (bf(R, D),), lambda q: ops.qprep_fwd(q, u, v, 0.125), R * D * 6)

# CTC at the bench's shape: T' = 875 frames max, U = 120 labels, V = 5004
V, Tc, U = 5004, 875, 120
Vp = (V + 7) // 8 * 8
in_l = torch.full((B,), Tc, device=dev, dtype=torch.int32)
tg_l = torch.full((B,), U, device=dev, dtype=torch.int32)
tg = torch.randint(4, V, (B, U), device=dev, dtype=torch.int32)
timed("ctc_loss (prep+scan+grad) B=24,T=875", lambda: (bf(B, Tc, Vp),),
      lambda lg: ops.ctc_loss(lg, V, in_l, tg, tg_l, 0), B * Tc * Vp * 4, nsets=3)
