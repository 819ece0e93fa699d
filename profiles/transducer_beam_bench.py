"""Transducer beam search at the recipes' decode shape: the host AdaptiveExpansionSearch (one utterance at a time)
against the batched device search (BatchedAdaptiveExpansionSearch), on the same random model.

Shape (examples/asr_librispeech/run_transformer_transducer.sh:263-265): 2 x 512 LSTM predictor, J = 512, V = 5004,
24 utterances x 250 encoder frames (10 s after 4x subsampling), beam 5, 20 expansions per frame, beta 2, gamma 2.3,
alpha 1, temperature 1.3; optionally a 4 x 800 LSTM LM at weight 0.4.  The encoder is not run: its joint-space
projections are random.  A random joint rarely emits blank, so every frame runs all 20 rounds (the worst case);
--blank-bias adds a constant to the blank logit; at 2.5 the 1-best carries about 0.16 tokens per frame.

Prints one JSON line per configuration: median ms per batch over --runs runs (CUDA events), tokens per frame,
native launches and host syncs per frame, peak memory, and whether the two searches agree."""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from espresso_b200 import lib, ops
from espresso_b200.tools.transducer_beam_search_decoder import AdaptiveExpansionSearch, BatchedAdaptiveExpansionSearch


def model(V, J, H, L, seed, lm_H=0, lm_L=0):
    g = torch.Generator().manual_seed(seed)

    def w(*shape, s=None):
        return (torch.randn(*shape, generator=g) * (s or shape[-1] ** -0.5)).cuda().bfloat16()

    p = dict(emb=w(V, H, s=1.0), Wih=[w(4 * H, H) for _ in range(L)], Whh=[w(4 * H, H) for _ in range(L)],
             b=[w(4 * H, s=0.1) for _ in range(L)], proj=w(J, H), W=w(V, J), bias=w(V, s=0.1))
    if lm_L:
        p.update(lemb=w(V, lm_H, s=1.0), lWih=[w(4 * lm_H, lm_H) for _ in range(lm_L)],
                 lWhh=[w(4 * lm_H, lm_H) for _ in range(lm_L)], lb=[w(4 * lm_H, s=0.1) for _ in range(lm_L)], lout=w(V, lm_H))
    return p


def cells(x, hs, cs, Wih, Whh, b):
    nh, nc = [], []
    for i in range(len(Wih)):
        gates = ops.linear(x, Wih[i], b[i]).float() + ops.linear(hs[:, i].contiguous(), Whh[i]).float()
        i_, f_, g_, o_ = gates.chunk(4, dim=1)
        c = torch.sigmoid(f_) * cs[:, i] + torch.sigmoid(i_) * torch.tanh(g_)
        x = (torch.sigmoid(o_) * torch.tanh(c)).bfloat16()
        nh.append(x)
        nc.append(c)
    return x, torch.stack(nh, 1), torch.stack(nc, 1)


def callbacks(p, pe, blank, blank_bias, H, L, lm_H, lm_L):
    """Batched callbacks over pe [B*T, J]; frame = b * T + t."""
    def joint_logits(frame, pd):
        n = pd.size(0)
        f = ops.joint_fwd(ops.gather_rows(pe, frame).view(n, 1, -1), pd.contiguous().view(n, 1, -1))
        lg = ops.linear(f.view(n, -1), p["W"], p["bias"])
        if blank_bias:
            lg[:, blank] += blank_bias
        return lg

    cb = dict(init_state=lambda n: (torch.zeros(n, L, H, device="cuda").bfloat16(), torch.zeros(n, L, H, device="cuda")),
              pred_step=lambda prev, hs, cs: cells(p["emb"][prev], hs, cs, p["Wih"], p["Whh"], p["b"]),
              project=lambda out: ops.linear(out, p["proj"]), joint_logits=joint_logits)
    if lm_L:
        cb.update(lm_init_state=lambda n: (torch.zeros(n, lm_L, lm_H, device="cuda").bfloat16(),
                                           torch.zeros(n, lm_L, lm_H, device="cuda")),
                  lm_step=lambda prev, hs, cs: cells(p["lemb"][prev], hs, cs, p["lWih"], p["lWhh"], p["lb"]),
                  lm_logits=lambda feat: ops.linear(feat.contiguous(), p["lout"]))
    return cb


def host_callbacks(cb, b, T, temperature):
    """One utterance's callbacks for AdaptiveExpansionSearch (joint_lprobs at frame t of utterance b)."""
    def joint_lprobs(t, out):
        n = out.size(0)
        frame = torch.full((n,), b * T + t, dtype=torch.int32, device="cuda")
        return torch.log_softmax(cb["joint_logits"](frame, cb["project"](out)).float() / temperature, dim=-1)

    h = dict(cb, joint_lprobs=joint_lprobs)
    if "lm_logits" in cb:
        h["lm_lprobs"] = lambda feat: torch.log_softmax(cb["lm_logits"](feat).float(), dim=-1)
    return h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=24)
    ap.add_argument("--T", type=int, default=250)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--host-runs", type=int, default=1)
    ap.add_argument("--host-utts", type=int, default=2, help="utterances the host search times (its ms scale per utterance)")
    ap.add_argument("--lm", action="store_true")
    ap.add_argument("--blank-bias", type=float, default=0.0)
    a = ap.parse_args()
    V, J, H, L, beam, E, beta, gamma, alpha, temp = 5004, 512, 512, 2, 5, 20, 2, 2.3, 1, 1.3
    lm_H, lm_L = (800, 4) if a.lm else (0, 0)
    p = model(V, J, H, L, 0, lm_H, lm_L)
    pe = (torch.randn(a.B * a.T, J, generator=torch.Generator().manual_seed(1)) * 0.5).cuda().bfloat16()
    cb = callbacks(p, pe, 0, a.blank_bias, H, L, lm_H, lm_L)
    core = AdaptiveExpansionSearch(V, 0, 1, 2, 2, beam, E, beta, gamma, alpha, True, False, 0.4, False)
    dev = BatchedAdaptiveExpansionSearch(core, temp)
    n_frames = torch.full((a.B,), a.T, dtype=torch.int32)

    syncs = [0]
    real_sync = torch.cuda.Stream.synchronize

    def counted_sync(self):
        syncs[0] += 1
        return real_sync(self)

    def timed(fn, runs):
        ms = []
        for _ in range(runs):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            out = fn()
            e.record()
            torch.cuda.synchronize()
            ms.append(s.elapsed_time(e))
        return statistics.median(ms), out

    with torch.no_grad():
        dev_fn = lambda: dev.search(n_frames, a.T, cb, torch.device("cuda"), use_lm=a.lm)  # noqa: E731
        dev_fn()  # warm-up
        torch.cuda.reset_peak_memory_stats()
        base_mem = torch.cuda.memory_allocated()
        n0 = lib.launch_count()
        torch.cuda.Stream.synchronize = counted_sync
        t0 = time.perf_counter()
        res = dev_fn()
        torch.cuda.synchronize()
        torch.cuda.Stream.synchronize = real_sync
        wall1 = time.perf_counter() - t0
        launches = lib.launch_count() - n0
        peak = torch.cuda.max_memory_allocated() - base_mem
        dev_ms, res = timed(dev_fn, a.runs)
        tokens_per_frame = sum(int((r[0][0] != 1).sum()) for r in res) / (a.B * a.T)

        hcb = [host_callbacks(cb, b, a.T, temp) for b in range(a.host_utts)]
        host_ms, host_res = timed(lambda: [core.search(a.T, hcb[b], torch.device("cuda"), use_lm=a.lm) for b in range(a.host_utts)],
                                  a.host_runs)
        agree = all(torch.equal(host_res[b][0].cpu(), res[b][0].cpu()) for b in range(a.host_utts))
        gpu = torch.cuda.get_device_name()
    print(json.dumps(dict(
        lm=a.lm, blank_bias=a.blank_bias, B=a.B, T=a.T, gpu=gpu,
        device_ms_per_batch=round(dev_ms, 1), host_ms_per_batch_extrapolated=round(host_ms / a.host_utts * a.B, 1),
        host_ms_per_utt=round(host_ms / a.host_utts, 1), speedup=round(host_ms / a.host_utts * a.B / dev_ms, 1),
        native_launches_per_frame=round(launches / a.T, 1), host_syncs_per_frame=round(syncs[0] / a.T, 2),
        tokens_per_frame=round(tokens_per_frame, 3), peak_search_mem_mb=round(peak / 2 ** 20, 1),
        device_wall_s_first_timed=round(wall1, 2), host_top_tokens_agree=agree)))


if __name__ == "__main__":
    main()
