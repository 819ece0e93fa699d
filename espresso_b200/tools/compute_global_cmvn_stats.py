"""Global CMVN statistics of a set of utterances -- what `OnTheFlyFbank.from_npz(global_cmvn_stats_path)` reads
(espresso/tools/compute_global_cmvn_stats.py:52-129 writes the same `gcmvn.npz` with keys `mean`, `std`; consumed by
fairseq/data/audio/feature_transforms/global_cmvn.py:20-29).

The reference computes fbank features per utterance on CPU threads and merges per-utterance sums / unnormalised variances
(the Lhotse pooling formula).  Here the features come from the device front end (`esp_frontend_fbank`, fp32 output, no CMVN,
no masking) batch by batch, and the per-bin sums of x and x^2 over the valid frames are accumulated in float64:
mean = S1 / n, std = sqrt(S2 / n - mean^2) -- the same population statistics the pooling formula yields.

    python -m espresso_b200.tools.compute_global_cmvn_stats wav.scp out_dir [--max-num-utts N] [--batch-seconds 600]

`wav.scp` lines: `<utt-id> <path to a WAVE or FLAC file>` (piped commands are a data-prep concern and not supported
here); FLAC files are uploaded compressed and decoded on the device."""
import argparse
import os

import numpy as np
import torch

from .. import ops as _ops
from ..data import flac as _flac
from ..data.audio_io import get_waveform


def global_cmvn_stats(waveforms, device, batch_seconds=600.0, sample_rate=16000):
    """waveforms: iterable of 1-D float32 arrays in int16 range (what get_waveform(..., normalization=False) returns) or
    of FlacStreams (espresso_b200.data.flac), which are batched compressed and decoded on the device.
    Returns (mean float64 [80], std float64 [80], number of frames)."""
    s1 = torch.zeros(80, dtype=torch.float64, device=device)
    s2 = torch.zeros(80, dtype=torch.float64, device=device)
    n_frames = 0
    batch, budget = [], 0

    def flush():
        nonlocal n_frames, batch, budget
        if not batch:
            return
        if isinstance(batch[0], _flac.FlacStream):
            wv, n = _flac.to_device(_flac.pack(batch, min_width=400), device)
        else:
            n = np.array([len(w) for w in batch], dtype=np.int32)
            wv = np.zeros((len(batch), max(int(n.max()), 400)), dtype=np.float32)
            for b, w in enumerate(batch):
                wv[b, : len(w)] = w
            wv, n = torch.from_numpy(wv).to(device), torch.from_numpy(n).to(device)
        feats, lens = _ops.frontend_fbank(wv, n, out_dtype=torch.float32)
        valid = (torch.arange(feats.shape[1], device=feats.device)[None, :] < lens[:, None].to(feats.device)).unsqueeze(-1)
        x = feats.double() * valid
        s1.add_(x.sum((0, 1)))
        s2.add_((x * x).sum((0, 1)))
        n_frames += int(lens.sum())
        batch, budget = [], 0

    for w in waveforms:
        if isinstance(w, _flac.FlacStream):
            if batch and not isinstance(batch[0], _flac.FlacStream):
                flush()
            n = w.total_samples
        else:
            if batch and isinstance(batch[0], _flac.FlacStream):
                flush()
            w = np.asarray(w, dtype=np.float32).reshape(-1)
            n = len(w)
        batch.append(w)
        budget += n
        if budget >= batch_seconds * sample_rate:
            flush()
    flush()
    if n_frames == 0:
        raise ValueError("no frames: every utterance is shorter than one 25 ms window")
    mean = s1 / n_frames
    std = torch.sqrt(torch.clamp(s2 / n_frames - mean * mean, min=0.0))
    return mean.cpu().numpy(), std.cpu().numpy(), n_frames


def main(argv=None):
    ap = argparse.ArgumentParser(description="Compute global CMVN stats (fbank80) with the device front end")
    ap.add_argument("file", help="lines '<utt-id> <wave file>'")
    ap.add_argument("output_dir")
    ap.add_argument("--max-num-utts", type=int, default=None)
    ap.add_argument("--batch-seconds", type=float, default=600.0)
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args(argv)

    def waves():
        with open(args.file, "r", encoding="utf-8") as f:
            for i, line in enumerate(f):
                if args.max_num_utts is not None and i == args.max_num_utts:
                    break
                _, path = line.rstrip().split(None, 1)
                if path.endswith("|"):
                    raise ValueError("piped commands are not supported here: decode to WAVE files first (%s)" % path)
                if path.lower().endswith(".flac"):  # decoded on the device, batch by batch
                    with open(path, "rb") as f:
                        w = _flac.read_stream(f.read())
                    sr = w.info.sample_rate
                else:
                    w, sr = get_waveform(path, normalization=False, always_2d=False)
                if sr != 16000:
                    raise ValueError("%s: %d Hz (the front end is built for 16 kHz)" % (path, sr))
                yield w

    mean, std, n = global_cmvn_stats(waves(), torch.device(args.device), args.batch_seconds)
    os.makedirs(args.output_dir, exist_ok=True)
    out = os.path.join(args.output_dir, "gcmvn.npz")
    with open(out, "wb") as f:
        np.savez(f, mean=mean, std=std)
    print("saved %s (%d frames)" % (out, n))


if __name__ == "__main__":
    main()
