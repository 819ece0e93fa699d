"""Device FLAC decoding (esp_flac_decode) on a LibriSpeech-shaped batch: 24 utterances of about 12 s, 16 kHz mono 16-bit.

Two batches: the LibriSpeech fixture (real libFLAC output, 11.9 s) tiled 24 times, and 24 synthetic utterances of 12 s
written by the test encoder at flac -5-like settings (blocks of 4096, LPC order 8, Rice partitions of order 4).  For
each: device time per batch (CUDA events around back-to-back decodes, status not read back), the upload of the packed
buffer (pinned, one copy) against the float32 waveform the WAVE path uploads, launches per batch, and a per-kernel split
from torch.profiler in a separate pass.  Every decoded batch is checked against the numpy decoder first.

    python profiles/flac_bench.py [--reps 50] [--out results/flac_bench.json]"""
import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_label():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the label is informative only
        return "unknown (%s)" % e


def batches():
    from flac_util import librispeech_like, speech_like

    with open(os.path.join(ROOT, "tests", "golden", "librispeech_6313-76958-0021.flac"), "rb") as f:
        fixture = f.read()
    rs = np.random.RandomState(0)
    synth = [librispeech_like(speech_like(rs, 192000)) for _ in range(4)]
    return {"fixture x24": [fixture] * 24, "encoder flac-5-like x24": [synth[i % 4] for i in range(24)]}


def time_batch(bufs, reps, dev):
    from espresso_b200 import lib, ops
    from espresso_b200.data import flac as FL
    from oracle import flac as F

    p = FL.pack([FL.read_stream(b) for b in bufs])
    t = p.buffer.to(dev)
    params, offsets, frames = p.views(t)
    out, st = ops.flac_decode(frames, offsets, params, p.width, p.max_channels, check=True)
    ref = {}
    for i, b in enumerate(bufs):
        if b not in ref:
            info, pcm, _ = F.decode(b)
            ref[b] = F.waveform(pcm, info["bps"])
        assert torch.equal(out[i, : len(ref[b])].cpu(), torch.from_numpy(ref[b])), "decode mismatch in row %d" % i
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    ops.flac_decode(frames, offsets, params, p.width, p.max_channels, check=False)
    torch.cuda.synchronize()
    launches = lib.launch_count() - n0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        ops.flac_decode(frames, offsets, params, p.width, p.max_channels, check=False)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        ops.flac_decode(frames, offsets, params, p.width, p.max_channels, check=False)
    e1.record()
    torch.cuda.synchronize()
    dec_ms = e0.elapsed_time(e1) / reps
    # the upload: packed buffer vs the float32 waveform of the same batch, both from pinned memory
    wave = torch.zeros(len(bufs), p.width, dtype=torch.float32).pin_memory()

    def h2d_ms(src):
        dst = torch.empty_like(src, device=dev)
        dst.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            dst.copy_(src, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    up_flac, up_wave = h2d_ms(p.buffer), h2d_ms(wave)
    samples = int(p.lengths.sum())
    # per-kernel device time, in a pass of its own
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            ops.flac_decode(frames, offsets, params, p.width, p.max_channels, check=False)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        m = re.search(r"flac_\w+_kernel", ev.key)
        if m:
            kernels[m.group(0)] = round(kernels.get(m.group(0), 0.0) + ev.device_time_total / 10.0 / 1e3, 4)
    return {"utterances": len(bufs), "audio_s": samples / 16000.0, "width": p.width,
            "decode_ms_per_batch": dec_ms, "launches_per_batch": launches, "kernel_ms_per_batch": kernels,
            "upload_bytes": p.buffer.numel(), "upload_bytes_float32_wave": wave.numel() * 4,
            "bytes_ratio": wave.numel() * 4 / p.buffer.numel(), "bytes_per_sample": p.buffer.numel() / samples,
            "h2d_ms_packed": up_flac, "h2d_ms_float32_wave": up_wave}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "flac_bench measures on the GPU"
    from espresso_b200 import lib

    lib.load()
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_label(), "batches": {k: time_batch(v, args.reps, dev) for k, v in batches().items()}}
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
