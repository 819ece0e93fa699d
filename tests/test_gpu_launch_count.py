"""GPU: every C-ABI entry point adds exactly the kernels it launched to lib.launch_count().  bench.py reports launches per
step from that counter and Trainer adds a captured graph's count on every replay, so a launch that is skipped but
counted (or run but not counted) skews both.  Each case calls one entry point once under torch.profiler and compares the
counter's delta with the kernels the profiler saw, leaving out ATen's (the wrappers' own fills) and copies.  The cases
cover every branch that changes how many kernels an entry point runs, and pin that number."""
import os
import sys

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile, schedule

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

DEV = torch.device("cuda:0")


def _bf(*shape):
    return torch.randn(*shape, device=DEV).bfloat16()


def _i32(values):
    return torch.tensor(values, dtype=torch.int32, device=DEV)


def _profile_step(fn):
    """(launch_count delta, CUDA-side events) of one call, recorded as the profiler's active step after a warm-up step
    that runs the same call."""
    from espresso_b200 import lib

    events = []
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], schedule=schedule(wait=0, warmup=1, active=1),
                 on_trace_ready=lambda p: events.extend(e.name for e in p.events()
                                                        if e.device_type == torch.autograd.DeviceType.CUDA)) as prof:
        fn()
        torch.cuda.synchronize()
        prof.step()
        n0 = lib.launch_count()
        fn()
        torch.cuda.synchronize()
        counted = lib.launch_count() - n0
        prof.step()
    return counted, events


def _native_kernels(fn, attempts=3):
    """(launch_count delta, names of the non-ATen kernels that ran) of one call.  The step's own GPU annotation
    ("ProfilerStep#") marks a delivered GPU trace; the profiler now and then returns a cycle without any GPU events, and
    such a cycle is measured again."""
    for _ in range(attempts):
        counted, events = _profile_step(fn)
        if any(n.startswith("ProfilerStep") for n in events):
            return counted, [n for n in events if not n.startswith(("ProfilerStep", "Memcpy", "Memset")) and "at::" not in n]
    pytest.fail("torch.profiler delivered no GPU trace in %d attempts" % attempts)


# ---------------------------------------------------------------------------------------------------------- cases
# name -> (kernels launched, setup); setup() builds the inputs and returns the call to count.
def _gemm(M, N, K):
    from espresso_b200 import ops

    x, w = _bf(M, K), _bf(N, K)
    return lambda: ops.linear(x, w)


def _linear_wgrad():
    from espresso_b200 import ops

    dy, x = _bf(512, 128), _bf(512, 64)
    gw, gb = torch.zeros(128 * 64, device=DEV), torch.zeros(128, device=DEV)
    return lambda: ops.linear_wgrad(dy, x, gw, gb)


def _conv(kind, stride):
    from espresso_b200 import ops

    B, T, F, Cin, Cout = 2, 9, 7, 64, 64
    x, w = _bf(B, T, F, Cin), _bf(Cout, 3, 3, Cin)
    To, Fo = (T + stride[0] - 1) // stride[0], (F + stride[1] - 1) // stride[1]
    dy = _bf(B, To, Fo, Cout)
    if kind == "fwd":
        return lambda: ops.conv3x3_fwd(x, w, stride)
    if kind == "dgrad":
        return lambda: ops.conv3x3_dgrad(dy, w, (B, T, F, Cin), stride)
    dw = torch.zeros(Cout, 3, 3, Cin, device=DEV)
    return lambda: ops.conv3x3_wgrad(dy, x, dw, stride)


def _conv_c1(kind):
    from espresso_b200 import ops

    x, w, dy = _bf(2, 9, 80), _bf(64, 3, 3), _bf(2, 5, 40, 64)
    if kind == "fwd":
        return lambda: ops.conv3x3_fwd(x, w, (2, 2))
    dw = torch.zeros(64, 3, 3, device=DEV)
    return lambda: ops.conv3x3_wgrad(dy, x, dw, (2, 2))


def _frontend(masks):
    from espresso_b200 import ops

    B = 2
    wave = torch.randn(B, 4000, device=DEV) * 1000
    n = _i32([4000, 3000])
    fm = _i32([[[3, 5]], [[10, 4]]]) if masks else None  # (first bin / frame, width) per utterance
    tm = _i32([[[2, 4]], [[0, 0]]]) if masks else None
    return lambda: ops.frontend_fbank(wave, n, freq_masks=fm, time_masks=tm)


def _ctc(T, want_grad):
    import ctypes as C

    from espresso_b200 import lib, ops

    B, V = 2, 13
    targets, tgt_lens = _i32([[1, 2, 3], [4, 5, 0]]), _i32([3, 2])
    if T > 0:
        x, in_lens = _bf(B, T, 16), _i32([T, T - 1])
        return lambda: ops.ctc_loss(x, V, in_lens, targets, tgt_lens, 0, want_grad=want_grad)
    # no frames at all: through the C ABI, as torch gives an empty tensor no address; no frame is read from x or grad
    L = lib.load()
    x, grad, in_lens, loss = _bf(B, 1, 16), _bf(B, 1, 16), _i32([0, 0]), torch.empty(B, device=DEV)
    ws = torch.empty(int(L.esp_ctc_workspace_bytes(B, 0, 3)), dtype=torch.uint8, device=DEV)
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    return lambda: lib.check(L.esp_ctc_loss(p(x), 16, 16, V, B, 0, p(in_lens), p(targets), 3, p(tgt_lens), 0, 1, 1.0, p(loss),
                                            p(grad) if want_grad else None, p(ws), stream))


def _rnnt(want_grad):
    from espresso_b200 import ops

    B, T, U1, V = 2, 5, 3, 11
    x = _bf(B, T, U1, 16)
    t_lens, u_lens, targets = _i32([5, 4]), _i32([2, 1]), _i32([[1, 2], [3, 0]])
    return lambda: ops.rnnt_loss(x, V, t_lens, u_lens, targets, 0, want_grad=want_grad)


def _ctc_beam(stage):
    from espresso_b200 import ops

    B, T, V, K, beam = 2, 6, 12, 4, 3
    x, lens = _bf(B, T, 16), _i32([6, 4])
    frames = ops.ctc_beam_frames(x, V, lens, K, 0)
    ws = ops.ctc_beam_workspace(B, T, beam, DEV)
    if stage == "frames":
        return lambda: ops.ctc_beam_frames(x, V, lens, K, 0)
    ops.ctc_beam_search(x, V, lens, frames, beam, 10.0, 0, T, ws)
    if stage == "search":
        return lambda: ops.ctc_beam_search(x, V, lens, frames, beam, 10.0, 0, T, ws)
    return lambda: ops.ctc_beam_finalize(lens, T, V, beam, 2, ws)


def _layer_norm(kind, d):
    from espresso_b200 import ops

    R = 48
    x, g, b = _bf(R, d), _bf(d), _bf(d)
    if kind == "fwd":
        return lambda: ops.layer_norm_fwd(x, g, b)
    y, mean, rstd = ops.layer_norm_fwd(x, g, b)
    dy, dg, db = _bf(R, d), torch.zeros(d, device=DEV), torch.zeros(d, device=DEV)
    if kind == "bwd":
        return lambda: ops.layer_norm_bwd(dy, x, mean, rstd, g, dg, db)
    return lambda: ops.layer_norm_bwd(dy, x, mean, rstd, g, dg, db, next_drop=(0.1, 7, 1.0))


def _elementwise(kind):
    from espresso_b200 import ops

    x = _bf(40, 64)
    if kind == "colsum_wide":
        wide, acc = _bf(24, 4096 + 64), torch.zeros(4096 + 64, device=DEV)
        return lambda: ops.colsum(wide, acc)
    if kind == "colsum":
        acc = torch.zeros(64, device=DEV)
        return lambda: ops.colsum(x, acc)
    if kind == "dropout":
        return lambda: ops.dropout(x, 0.1, 3)
    if kind == "mask_rows":
        xm, lens = _bf(2, 20, 64), _i32([20, 11])
        return lambda: ops.mask_rows_(xm, lens)
    if kind == "qprep_fwd":
        u, v = _bf(64), _bf(64)
        return lambda: ops.qprep_fwd(x, u, v, 0.125)
    dq = _bf(40, 64)
    return lambda: ops.qprep_bwd(x, x, 0.125, dq)


def _softmax(kind):
    from espresso_b200 import ops

    H, B, T = 2, 2, 20
    scores = _bf(H, B, T, 24)
    lens = _i32([20, 13])
    if kind == "fwd":
        return lambda: ops.attn_softmax_fwd(scores, T, lens, drop_p=0.1, seed=5)
    p, _ = ops.attn_softmax_fwd(scores, T, lens)
    dp = _bf(H, B, T, 24)
    return lambda: ops.attn_softmax_bwd(p, dp, T, 40)


def _attn_fused(kind):
    from espresso_b200 import ops

    B, T, H, hd = 2, 16, 2, 64
    d = H * hd
    qkv = _bf(B * T, 3 * d)
    qu, qv, pos = _bf(B * T, d), _bf(B * T, d), _bf(2 * T - 1, d)
    lens = _i32([16, 9])
    if kind == "fwd":
        return lambda: ops.attn_fused_fwd(qu, qv, qkv[:, d:2 * d], qkv[:, 2 * d:], pos, B, T, H, lens)
    ctx, p, pd = ops.attn_fused_fwd(qu, qv, qkv[:, d:2 * d], qkv[:, 2 * d:], pos, B, T, H, lens)
    dctx, dqkv = _bf(B * T, d), _bf(B * T, 3 * d)
    ldp = (2 * T - 1 + 7) // 8 * 8
    return lambda: ops.attn_fused_bwd(dctx, ctx, qu, qkv[:, 2 * d:], p, pd, B, T, H, ldp, dqkv[:, d:2 * d], dqkv[:, 2 * d:])


def _conv_module(kind):
    from espresso_b200 import ops

    B, T, C, k = 2, 20, 64, 15
    g, w, dy = _bf(B, T, 2 * C), _bf(C, k), _bf(B, T, C)
    if kind == "glu_fwd":
        return lambda: ops.glu_dwconv_fwd(g, w)
    if kind == "glu_bwd":
        dw = torch.zeros(C, k, device=DEV)
        return lambda: ops.glu_dwconv_bwd(dy, g, w, dw)
    y, stats = ops.glu_dwconv_fwd(g, w)
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    if kind == "bn_stats":
        return lambda: ops.bn_stats(y, C)
    if kind == "bn_finalize":
        return lambda: ops.bn_finalize(stats, B * T, C, 1e-5, 0.1, rm, rv, True)
    mr = ops.bn_finalize(stats, B * T, C, 1e-5, 0.1, rm, rv, True)
    gamma, beta = _bf(C), _bf(C)
    if kind == "bn_act_fwd":
        return lambda: ops.bn_act_fwd(y, mr, gamma, beta)
    dg, db = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    return lambda: ops.bn_act_bwd(dy, y, mr, gamma, beta, dg, db)


def _optim(kind):
    from espresso_b200 import ops

    n = 1000
    g, out = torch.randn(n, device=DEV), torch.zeros(1, device=DEV)
    if kind == "sumsq":
        return lambda: ops.sumsq(g, out)
    if kind == "cast_f32_bf16":
        y = torch.empty(n, dtype=torch.bfloat16, device=DEV)
        return lambda: ops.cast_f32_bf16(g, y)
    if kind == "cast_bf16_f32":
        x, y = g.bfloat16(), torch.empty(n, device=DEV)
        return lambda: ops.cast_bf16_f32(x, y)
    ops.sumsq(g, out)
    p32, m, v = torch.randn(n, device=DEV), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    p16 = p32.bfloat16()
    return lambda: ops.adam_step(p32, m, v, g, p16, 1e-3, 0.9, 0.98, 1e-8, 0.0, 1, out)


def _decoder(kind):
    from espresso_b200 import ops

    V, U = 40, 6
    logits = _bf(2 * U, 48)
    tokens = torch.randint(4, V, (2 * U,), dtype=torch.int32, device=DEV)
    if kind == "lsce":
        return lambda: ops.lsce_loss(logits, V, tokens, 1, 0.1)
    E, pos = _bf(V, 64), _bf(U, 64)
    if kind == "embed_fwd":
        return lambda: ops.embed_fwd(tokens, E, pos, U, 8.0, 1)
    if kind == "embed_bwd":
        dx, dE = _bf(2 * U, 64), torch.zeros(V, 64, device=DEV)
        return lambda: ops.embed_bwd(tokens, dx, dE, 8.0, 1)
    return lambda: ops.argmax_rows(logits, V)


def _beam(kind):
    from espresso_b200 import ops

    bsz, beam, V, max_len = 2, 3, 20, 6
    N, L, K = bsz * beam, max_len + 2, 2 * beam
    cand, x, prev = torch.empty(N, V, device=DEV), _bf(N, 24), torch.zeros(N, device=DEV)
    if kind == "merge":
        return lambda: ops.beam_merge(x, V, True, cand, prev_scores=prev)
    ops.beam_merge(x, V, True, cand)
    if kind in ("topk", "topk_large"):
        k = K if kind == "topk" else 20
        return lambda: ops.beam_topk(cand, bsz, beam * V, beam * V, k, V)
    if kind == "gather_rows":
        src = _bf(N, 64)
        return lambda: ops.gather_rows(src, _i32([2, 0, 1, 5, 4, 3]))
    cs, ct, cb = ops.beam_topk(cand, bsz, beam * V, beam * V, K, V)

    class St:
        pass

    st = St()
    st.tokens, st.tokens_alt = (torch.full((N, L), 1, dtype=torch.int32, device=DEV) for _ in range(2))
    st.scores, st.scores_alt = (torch.zeros(N, L - 1, device=DEV) for _ in range(2))
    st.ignore, st.finished = torch.zeros(N, dtype=torch.uint8, device=DEV), torch.zeros(bsz, dtype=torch.uint8, device=DEV)
    st.nfin = torch.zeros(bsz, dtype=torch.int32, device=DEV)
    st.fin_tokens = torch.full((bsz, beam, L - 1), 1, dtype=torch.int32, device=DEV)
    st.fin_len = torch.zeros(bsz, beam, dtype=torch.int32, device=DEV)
    st.fin_score, st.fin_pos = torch.zeros(bsz, beam, device=DEV), torch.zeros(bsz, beam, L - 1, device=DEV)
    st.new_order, st.n_unfinished = torch.zeros(N, dtype=torch.int32, device=DEV), _i32([bsz])
    args = (0, max_len, bsz, beam, K, 2, 1, True, 1.0, cs, ct, cb, st)
    if kind == "bookkeep":
        return lambda: ops.beam_bookkeep(*args)
    Tk = 9
    st.fin_attn = torch.zeros(bsz, beam, L - 1, Tk, device=DEV)
    att, anc = torch.rand(max_len + 1, N, Tk, device=DEV), torch.zeros(max_len + 1, N, dtype=torch.int32, device=DEV)
    return lambda: ops.beam_bookkeep_attn(*args, att, anc)


def _decode_attn(kind):
    from espresso_b200 import ops

    bsz, beam, H, hd, Tk, T_max = 2, 3, 4, 16, 11, 5
    N, d = bsz * beam, H * hd
    q = _bf(N, d)
    if kind == "self":
        kvc, anc = _bf(T_max, N, 2 * d), torch.zeros(T_max, N, dtype=torch.int32, device=DEV)
        return lambda: ops.decode_self_attn(q, kvc, anc, 3, H, 0.25)
    if kind == "ancestry":
        a_in, a_out = torch.zeros(T_max, N, dtype=torch.int32, device=DEV), torch.empty(T_max, N, dtype=torch.int32, device=DEV)
        return lambda: ops.decode_update_ancestry(a_in, a_out, _i32([1, 0, 2, 5, 4, 3]), 2)
    kv, lens = _bf(bsz, Tk, 2 * d), _i32([11, 7])
    if kind == "cross":
        return lambda: ops.decode_cross_attn(q, kv, lens, beam, H, 0.25)
    w = torch.empty(N, Tk, device=DEV)
    return lambda: ops.decode_cross_attn_weights(q, kv, lens, beam, H, 0.25, w)


def _joint(kind):
    from espresso_b200 import ops

    enc, dec = _bf(2, 5, 64), _bf(2, 3, 64)
    if kind == "fwd":
        return lambda: ops.joint_fwd(enc, dec)
    f = ops.joint_fwd(enc, dec)
    df = _bf(*f.shape)
    return lambda: ops.joint_bwd(df, f)


def _lookahead(kind):
    from test_lookahead_lm import _dicts
    from espresso_b200 import ops
    from espresso_b200.tools.tensorized_prefix_tree import TensorizedPrefixTree

    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lookahead_lm.npz"))
    sub, wrd = _dicts(g)
    tree = TensorizedPrefixTree.build(wrd, sub)
    tr = tree.to(DEV)
    N, Vs, Vw = 6, len(sub), len(wrd)
    ld = (Vs + 7) // 8 * 8
    prev = torch.randint(0, Vs, (N,), dtype=torch.int32, device=DEV)
    nodes = torch.randint(0, tree.num_nodes, (N,), dtype=torch.int32, device=DEV)
    nodes_out, words = torch.zeros_like(nodes), torch.zeros_like(nodes)
    order = _i32([1, 0, 2, 5, 4, 3])
    if kind == "words":
        return lambda: ops.lookahead_words(nodes, order, tr["node_word"], wrd.unk(), nodes_out, words)
    wl = _bf(N, Vw)
    cum, cum_out, eos_lp = torch.rand(N, Vw, device=DEV), torch.empty(N, Vw, device=DEV), torch.empty(N, device=DEV)
    if kind == "cumsum":
        return lambda: ops.wordlm_cumsum(wl, Vw, prev, 1, sub.space(), False, cum, order, cum_out, eos_lp, wrd.eos())
    out = torch.zeros(N, ld, device=DEV)
    if kind == "step":
        root = torch.full((N,), 1, dtype=torch.int32, device=DEV)
        ops.wordlm_cumsum(wl, Vw, prev, 1, sub.space(), True, cum, None, cum_out, eos_lp, wrd.eos())
        return lambda: ops.lookahead_step(prev, 1, True, root, nodes_out, cum_out, Vw, eos_lp, tr, sub.space(), sub.eos(),
                                          sub.pad(), wrd.unk(), 0.0, True, 1e-10, out, Vs)
    wlp = torch.log_softmax(torch.randn(N, Vw, device=DEV), -1)
    sl, out_prev = _bf(N, ld), torch.randn(N, ld, device=DEV)
    cum_in, cum_new = torch.randn(N, device=DEV), torch.zeros(N, device=DEV)
    return lambda: ops.multilevel_step(prev, 1, False, nodes, nodes_out, order, wlp, Vw, sl, True, 0.7, out_prev, cum_in,
                                       cum_new, tr, sub.space(), sub.eos(), wrd.unk(), wrd.eos(), -1.7, True, -10.0, out, Vs)


CASES = {
    "gemm_mc1": (1, lambda: _gemm(64, 64, 64)),       # N <= 64: 64-wide tiles, single CTAs
    "gemm_mc2": (1, lambda: _gemm(256, 256, 128)),    # 128-wide tiles on an even tile count: 2-CTA multicast clusters
    "gemm_wgrad_rowsum": (1, _linear_wgrad),
    "conv3x3_fwd": (1, lambda: _conv("fwd", (1, 1))),
    "conv3x3_dgrad_stride1": (1, lambda: _conv("dgrad", (1, 1))),
    "conv3x3_dgrad_stride2": (4, lambda: _conv("dgrad", (2, 2))),  # one launch per output parity class
    "conv3x3_wgrad": (1, lambda: _conv("wgrad", (2, 2))),
    "conv3x3_c1_fwd": (1, lambda: _conv_c1("fwd")),
    "conv3x3_c1_wgrad": (1, lambda: _conv_c1("wgrad")),
    "frontend": (1, lambda: _frontend(False)),
    "frontend_masks": (2, lambda: _frontend(True)),    # + the SpecAugment paint kernel
    "ctc_loss": (3, lambda: _ctc(7, False)),
    "ctc_loss_grad": (4, lambda: _ctc(7, True)),
    "ctc_loss_t0": (2, lambda: _ctc(0, True)),         # no frames: neither prep nor grad runs
    "ctc_beam_frames": (1, lambda: _ctc_beam("frames")),
    "ctc_beam_search": (1, lambda: _ctc_beam("search")),
    "ctc_beam_finalize": (1, lambda: _ctc_beam("finalize")),
    "rnnt_loss": (3, lambda: _rnnt(False)),
    "rnnt_loss_grad": (4, lambda: _rnnt(True)),
    "joint_fwd": (1, lambda: _joint("fwd")),
    "joint_bwd": (1, lambda: _joint("bwd")),
    "layer_norm_fwd": (1, lambda: _layer_norm("fwd", 64)),
    "layer_norm_bwd": (1, lambda: _layer_norm("bwd", 64)),
    "layer_norm_bwd2": (1, lambda: _layer_norm("bwd2", 64)),
    "layer_norm_bwd2_wide": (1, lambda: _layer_norm("bwd2", 1024)),  # shared-memory opt-in above 48 KB
    "colsum": (1, lambda: _elementwise("colsum")),
    "colsum_wide": (2, lambda: _elementwise("colsum_wide")),  # more than 4096 columns: two column panels
    "dropout": (1, lambda: _elementwise("dropout")),
    "mask_rows": (1, lambda: _elementwise("mask_rows")),
    "qprep_fwd": (1, lambda: _elementwise("qprep_fwd")),
    "qprep_bwd": (1, lambda: _elementwise("qprep_bwd")),
    "attn_softmax_fwd": (1, lambda: _softmax("fwd")),
    "attn_softmax_bwd": (1, lambda: _softmax("bwd")),
    "attn_fused_fwd": (1, lambda: _attn_fused("fwd")),
    "attn_fused_bwd": (3, lambda: _attn_fused("bwd")),   # row dots, fused backward, skew
    "glu_dwconv_fwd": (1, lambda: _conv_module("glu_fwd")),
    "glu_dwconv_bwd": (1, lambda: _conv_module("glu_bwd")),
    "bn_stats": (1, lambda: _conv_module("bn_stats")),
    "bn_finalize": (1, lambda: _conv_module("bn_finalize")),
    "bn_act_fwd": (1, lambda: _conv_module("bn_act_fwd")),
    "bn_act_bwd": (3, lambda: _conv_module("bn_act_bwd")),  # reduce, parameter gradients, apply
    "sumsq": (1, lambda: _optim("sumsq")),
    "adam_step": (1, lambda: _optim("adam")),
    "cast_f32_bf16": (1, lambda: _optim("cast_f32_bf16")),
    "cast_bf16_f32": (1, lambda: _optim("cast_bf16_f32")),
    "lsce_loss": (1, lambda: _decoder("lsce")),
    "embed_fwd": (1, lambda: _decoder("embed_fwd")),
    "embed_bwd": (1, lambda: _decoder("embed_bwd")),
    "argmax_rows": (1, lambda: _decoder("argmax")),
    "beam_merge": (1, lambda: _beam("merge")),
    "beam_topk": (1, lambda: _beam("topk")),
    "beam_topk_large": (1, lambda: _beam("topk_large")),
    "beam_bookkeep": (1, lambda: _beam("bookkeep")),
    "beam_bookkeep_attn": (1, lambda: _beam("bookkeep_attn")),
    "gather_rows": (1, lambda: _beam("gather_rows")),
    "decode_self_attn": (1, lambda: _decode_attn("self")),
    "decode_cross_attn": (1, lambda: _decode_attn("cross")),
    "decode_cross_attn_weights": (1, lambda: _decode_attn("cross_weights")),
    "decode_update_ancestry": (1, lambda: _decode_attn("ancestry")),
    "lookahead_words": (1, lambda: _lookahead("words")),
    "wordlm_cumsum": (1, lambda: _lookahead("cumsum")),
    "lookahead_step": (1, lambda: _lookahead("step")),
    "multilevel_step": (1, lambda: _lookahead("multilevel")),
}


@pytest.mark.parametrize("name", list(CASES))
def test_launch_count_matches_kernels_run(name):
    expected, setup = CASES[name]
    torch.manual_seed(0)
    counted, ran = _native_kernels(setup())
    assert len(ran) == expected, (name, ran)
    assert counted == expected, (name, counted, ran)
