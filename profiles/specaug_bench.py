"""Time esp_specaug_features on a LibriSpeech-shaped 26 000-frame batch of 80-dim features, with the adaptive policy at
W = 0 (masks only) and W = 80 (time warp + masks), fp32 -> fp32 (Kaldi features) and fp32 -> bf16 (front end scratch ->
encoder input).  Two timings per case, both with CUDA events after `--warmup` calls:
  us_per_call: `--iters` back-to-back calls of ops.specaug_features from Python (host cost of the wrapper included);
  us_device:   replays of a CUDA graph holding 50 calls, i.e. the kernels' device time with the launches pre-recorded.
Prints one JSON line per case with the card's name and power limit and the bytes the algorithm moves (input frames read
once, the whole output written once) over us_device.  With --out the lines are also written to that file.

    python profiles/specaug_bench.py [--iters 2000] [--warmup 200] [--out specaug_bench.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from espresso_b200 import ops  # noqa: E402
from espresso_b200.data import specaugment as SA  # noqa: E402


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the timing does not depend on it
        q = "unknown (%s)" % e
    return q


def _batch(W, dev):
    rs = np.random.RandomState(0)
    lens = []
    while sum(lens) < 26000:
        lens.append(int(rs.randint(200, 1700)))
    lens.sort(reverse=True)
    B, T, F = len(lens), lens[0], 80
    x = torch.zeros(B, T, F)
    for b, m in enumerate(lens):
        x[b, :m] = torch.from_numpy(rs.randn(m, F).astype(np.float32))
    pol = SA.AdaptiveSpecAugmentConfig.from_config_dict(
        {"time_warp_W": W, "freq_mask_F": 27, "freq_mask_N": 2, "time_mask_pm": 0.04, "time_mask_ps": 0.04})
    draws = []
    for b, m in enumerate(lens):
        with SA.numpy_seed(1, 1, b):
            draws.append(SA.draw_specaugment(pol, m, F))
    fm, tm = SA.pack_masks([d[1] for d in draws], [d[2] for d in draws])
    warp = torch.from_numpy(SA.pack_warps([d[0] for d in draws])).to(dev) if W > 0 else None
    return (x.to(dev), torch.tensor(lens, dtype=torch.int32, device=dev), warp, torch.from_numpy(fm).to(dev),
            torch.from_numpy(tm).to(dev), lens)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("specaug_bench needs a GPU")
    dev = torch.device("cuda:0")
    card = _card()
    rows = []
    for W in (0, 80):
        x, lens, warp, fm, tm, lens_host = _batch(W, dev)
        for out_dtype in (torch.float32, torch.bfloat16):
            call = lambda: ops.specaug_features(x, lens, warp, fm, tm, out_dtype=out_dtype)  # noqa: E731
            for _ in range(a.warmup):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.iters):
                call()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / a.iters
            g = torch.cuda.CUDAGraph()
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                call()
                torch.cuda.synchronize()
                with torch.cuda.graph(g, stream=s):
                    for _ in range(50):
                        call()
            torch.cuda.current_stream().wait_stream(s)
            for _ in range(5):
                g.replay()
            torch.cuda.synchronize()
            reps = max(1, a.iters // 50)
            e0.record()
            for _ in range(reps):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            us_dev = e0.elapsed_time(e1) * 1e3 / (reps * 50)
            B, T, F = x.shape
            moved = sum(lens_host) * F * 4 + B * T * F * (4 if out_dtype == torch.float32 else 2)
            row = {"card": card, "W": W, "out": str(out_dtype).split(".")[-1], "B": B, "T": T, "frames": sum(lens_host),
                   "us_per_call": round(us, 2), "us_device": round(us_dev, 2), "bytes": moved,
                   "GB_per_s": round(moved / us_dev / 1e3, 1)}
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
