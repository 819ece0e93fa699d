"""FLAC input on the host side of the device decoder (csrc/flac.cu, esp_flac_decode).

LibriSpeech ships FLAC, and the reference reads it per utterance through libsndfile (fairseq/data/audio/audio_utils.py:
69-126).  Here the host only parses the metadata and keeps the compressed frames; a batch goes up to the device as ONE
pinned buffer (about 1.1 bytes per sample for LibriSpeech instead of 4 for float32 PCM) and is decoded there, before the
Trainer: the model, its CUDA-graph buckets (keyed on the waveform shape) and SpecAugment see the same float32 [B, N]
waveform a WAVE batch gives.

    info = read_info(fp)                        # STREAMINFO of an open binary file (seekable), or ValueError
    s = read_stream(buf)                        # FlacStream: parameters + the bytes from the first frame on
    packed = pack([s, ...], names=utt_ids)      # PackedFlac: one uint8 buffer (params | offsets | frames)
    src_tokens, src_lengths = to_device(packed, "cuda:0")"""
import io
import struct
from dataclasses import dataclass

import numpy as np
import torch

_PARAMS = 5  # int64 per stream in the packed buffer: total samples, sample rate, channels, bps, max block size


@dataclass
class FlacInfo:
    sample_rate: int
    channels: int
    bps: int
    total_samples: int
    md5: bytes
    min_blocksize: int
    max_blocksize: int
    first_frame: int  # byte offset of the first frame (after the last metadata block)


@dataclass
class FlacStream:
    info: FlacInfo
    frames: bytes  # the stream from its first frame on

    @property
    def total_samples(self):
        return self.info.total_samples


def _read_exact(fp, n):
    b = fp.read(n)
    if len(b) != n:
        raise ValueError("truncated FLAC stream")
    return b


def read_info(fp):
    """Parse the fLaC marker and the metadata blocks of an open binary file; returns FlacInfo.  STREAMINFO must come
    first (RFC 9639 section 8.1); other blocks are skipped up to the one with the last-block flag.  Raises ValueError
    for anything the device decoder does not take: a bad marker, truncation, no STREAMINFO, 32-bit samples (libsndfile
    does not read them either), fewer than 4 bits, or an unknown (zero) total sample count."""
    if fp.read(4) != b"fLaC":
        raise ValueError("not a FLAC stream (no fLaC marker)")
    pos, info = 4, None
    while True:
        hdr = _read_exact(fp, 4)
        last, btype, n = hdr[0] >> 7, hdr[0] & 0x7F, int.from_bytes(hdr[1:], "big")
        if btype == 0 and info is None and n >= 34:
            b = _read_exact(fp, n)
            minbs, maxbs = struct.unpack(">HH", b[:4])
            v = int.from_bytes(b[10:18], "big")
            info = FlacInfo(sample_rate=v >> 44, channels=((v >> 41) & 7) + 1, bps=((v >> 36) & 31) + 1,
                            total_samples=v & ((1 << 36) - 1), md5=bytes(b[18:34]), min_blocksize=minbs, max_blocksize=maxbs,
                            first_frame=0)
        elif info is None:
            raise ValueError("FLAC stream without STREAMINFO as its first metadata block")
        else:
            _read_exact(fp, n)  # skipped block; reading (not seeking) also detects truncation
        pos += 4 + n
        if last:
            break
    info.first_frame = pos
    if info.bps == 32 or info.bps < 4:
        raise ValueError("FLAC with %d bits per sample is not supported (4 to 24 bits)" % info.bps)
    if info.total_samples == 0:
        raise ValueError("FLAC stream with an unknown total sample count")
    return info


def is_flac(buf):
    return bytes(buf[:4]) == b"fLaC"


def read_stream(buf):
    """bytes of a whole .flac file -> FlacStream."""
    info = read_info(io.BytesIO(buf))
    if len(buf) <= info.first_frame:
        raise ValueError("FLAC stream without frames")
    return FlacStream(info, bytes(buf[info.first_frame:]))


@dataclass
class PackedFlac:
    """A batch of streams in one uint8 buffer: int64 params [B, 5] | int64 offsets [B + 1] | frames, pinned when CUDA is
    available.  `width` is the decoded row length N, `lengths` the int32 sample counts."""
    buffer: torch.Tensor
    batch: int
    width: int
    max_channels: int
    lengths: torch.Tensor
    names: list = None

    def views(self, t):
        """(params, offsets, frames) views of `t`, a copy of `buffer` (on any device)."""
        B = self.batch
        head = 8 * (_PARAMS * B + B + 1)
        params = t[: 8 * _PARAMS * B].view(torch.int64).view(B, _PARAMS)
        return params, t[8 * _PARAMS * B: head].view(torch.int64), t[head:]


def pack(streams, names=None, pad_to_multiple=1, min_width=0):
    """FlacStreams -> PackedFlac whose decoded rows are max(total samples) long (rounded up to pad_to_multiple, at least
    min_width), like collate_frames pads WAVE batches."""
    B = len(streams)
    totals = [s.info.total_samples for s in streams]
    width = max(max(totals), min_width)
    if pad_to_multiple > 1:
        width = (width + pad_to_multiple - 1) // pad_to_multiple * pad_to_multiple
    params = np.array([[s.info.total_samples, s.info.sample_rate, s.info.channels, s.info.bps, s.info.max_blocksize]
                       for s in streams], dtype=np.int64).reshape(B, _PARAMS)
    offsets = np.zeros(B + 1, dtype=np.int64)
    offsets[1:] = np.cumsum([len(s.frames) for s in streams])
    head = params.tobytes() + offsets.tobytes()
    buf = torch.empty(len(head) + int(offsets[-1]), dtype=torch.uint8,
                      pin_memory=torch.cuda.is_available())
    arr = buf.numpy()
    arr[: len(head)] = np.frombuffer(head, dtype=np.uint8)
    for s, o in zip(streams, offsets[:-1]):
        arr[len(head) + o: len(head) + o + len(s.frames)] = np.frombuffer(s.frames, dtype=np.uint8)
    return PackedFlac(buffer=buf, batch=B, width=int(width), max_channels=max(s.info.channels for s in streams),
                      lengths=torch.tensor(totals, dtype=torch.int32), names=names)


def to_device(packed, device):
    """Upload the packed batch (one copy) and decode it on the device -> (src_tokens float32 [B, width] in int16 range,
    zero past each length, src_lengths int32 [B] in samples).  Raises RuntimeError naming a failing utterance."""
    from .. import ops as _ops

    dev = torch.device(device)
    t = packed.buffer.to(dev, non_blocking=True)
    params, offsets, frames = packed.views(t)
    out, _ = _ops.flac_decode(frames, offsets, params, packed.width, packed.max_channels, names=packed.names)
    return out, packed.lengths.to(dev, non_blocking=True)
