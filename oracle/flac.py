"""Oracle: a plain FLAC decoder written from RFC 9639 (numpy + Python integers), with the header CRC-8, the frame CRC-16
and the STREAMINFO MD5 checks.  It is the reference the device decoder (csrc/flac.cu) is compared against, bit for bit.

    info, pcm = decode(buf)      # pcm: int64 [channels, total_samples]; raises ValueError on any malformed input
    wav = waveform(pcm, bps)     # float32 [total_samples]: s / 2^(bps-1) * 2^15, channels averaged in float32

It walks the stream frame by frame from the first frame (no sync search): every frame must start where the previous one
ended, carry the next sample number and pass both CRCs, and the frames must cover STREAMINFO's total exactly."""
import hashlib
import struct

import numpy as np


def _crc_table(poly, width):
    top, mask, out = 1 << (width - 1), (1 << width) - 1, []
    for b in range(256):
        c = b << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) if c & top else (c << 1)
        out.append(c & mask)
    return out


_CRC8 = _crc_table(0x07, 8)
_CRC16 = _crc_table(0x8005, 16)


def crc8(data):
    c = 0
    for b in data:
        c = _CRC8[c ^ b]
    return c


def crc16(data):
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ _CRC16[(c >> 8) ^ b]
    return c


class Bits:
    """MSB-first bit reader over a bytes object; reading past the end raises ValueError."""

    def __init__(self, buf, pos_bytes=0):
        self.buf, self.pos, self.limit = buf, pos_bytes * 8, len(buf) * 8

    def u(self, n):
        if n == 0:
            return 0
        if self.pos + n > self.limit:
            raise ValueError("truncated frame")
        i, sh = self.pos >> 3, self.pos & 7
        nb = (sh + n + 7) >> 3
        v = int.from_bytes(self.buf[i: i + nb], "big")
        self.pos += n
        return (v >> (nb * 8 - sh - n)) & ((1 << n) - 1)

    def s(self, n):
        v = self.u(n)
        return v - (1 << n) if n and v >> (n - 1) else v

    def unary(self):
        """Number of 0 bits before the next 1 bit (consumed)."""
        q = 0
        while True:
            if self.pos >= self.limit:
                raise ValueError("truncated frame")
            i, sh = self.pos >> 3, self.pos & 7
            b = self.buf[i] & (0xFF >> sh)
            if b:
                z = 8 - b.bit_length() - sh
                self.pos += z + 1
                return q + z
            q += 8 - sh
            self.pos += 8 - sh


BLOCK_SIZES = {1: 192, 2: 576, 3: 1152, 4: 2304, 5: 4608, **{c: 256 << (c - 8) for c in range(8, 16)}}
SAMPLE_RATES = {1: 88200, 2: 176400, 3: 192000, 4: 8000, 5: 16000, 6: 22050, 7: 24000, 8: 32000, 9: 44100, 10: 48000,
                11: 96000}
BPS = {1: 8, 2: 12, 4: 16, 5: 20, 6: 24, 7: 32}


def parse_streaminfo(buf):
    """-> dict(sample_rate, channels, bps, total_samples, md5, min_blocksize, max_blocksize, first_frame)."""
    if len(buf) < 4 or buf[:4] != b"fLaC":
        raise ValueError("not a FLAC stream")
    pos, info = 4, None
    while True:
        if pos + 4 > len(buf):
            raise ValueError("truncated metadata")
        last, btype, n = buf[pos] >> 7, buf[pos] & 0x7F, int.from_bytes(buf[pos + 1: pos + 4], "big")
        if pos + 4 + n > len(buf):
            raise ValueError("truncated metadata")
        if btype == 0:
            b = buf[pos + 4: pos + 4 + 34]
            minbs, maxbs = struct.unpack(">HH", b[:4])
            v = int.from_bytes(b[10:18], "big")
            info = dict(min_blocksize=minbs, max_blocksize=maxbs, sample_rate=v >> 44, channels=((v >> 41) & 7) + 1,
                        bps=((v >> 36) & 31) + 1, total_samples=v & ((1 << 36) - 1), md5=bytes(b[18:34]))
        elif info is None:
            raise ValueError("the first metadata block is not STREAMINFO")
        pos += 4 + n
        if last:
            break
    info["first_frame"] = pos
    return info


def _utf8(buf, pos):
    b0 = buf[pos]
    if b0 < 0x80:
        return b0, pos + 1
    n = 8 - (b0 ^ 0xFF).bit_length()  # leading ones
    if n < 2 or n > 7:
        raise ValueError("bad coded number")
    v = b0 & (0x7F >> n)
    for k in range(1, n):
        c = buf[pos + k]
        if c & 0xC0 != 0x80:
            raise ValueError("bad coded number")
        v = (v << 6) | (c & 0x3F)
    return v, pos + n


def parse_header(buf, pos, info):
    """Frame header at byte `pos` -> dict(bs, first_sample, assign, channels, bps, end).  ValueError if it is not a
    header of this stream (bad sync, reserved codes, parameters differing from STREAMINFO, CRC-8)."""
    if pos + 4 > len(buf) or buf[pos] != 0xFF or buf[pos + 1] & 0xFE != 0xF8:
        raise ValueError("no frame sync")
    variable = buf[pos + 1] & 1
    bsc, src = buf[pos + 2] >> 4, buf[pos + 2] & 15
    assign, bpsc, res = buf[pos + 3] >> 4, (buf[pos + 3] >> 1) & 7, buf[pos + 3] & 1
    if bsc == 0 or src == 15 or assign > 10 or bpsc == 3 or res:
        raise ValueError("reserved code in frame header")
    num, p = _utf8(buf, pos + 4)
    if bsc == 6:
        bs, p = buf[p] + 1, p + 1
    elif bsc == 7:
        bs, p = int.from_bytes(buf[p: p + 2], "big") + 1, p + 2
    else:
        bs = BLOCK_SIZES[bsc]
    if src == 12:
        rate, p = buf[p] * 1000, p + 1
    elif src == 13:
        rate, p = int.from_bytes(buf[p: p + 2], "big"), p + 2
    elif src == 14:
        rate, p = int.from_bytes(buf[p: p + 2], "big") * 10, p + 2
    else:
        rate = SAMPLE_RATES.get(src, info["sample_rate"])
    if p >= len(buf) or crc8(buf[pos:p]) != buf[p]:
        raise ValueError("frame header CRC-8 mismatch")
    bps = BPS.get(bpsc, info["bps"])
    channels = assign + 1 if assign < 8 else 2
    if bps != info["bps"] or channels != info["channels"] or rate != info["sample_rate"] or bs > info["max_blocksize"]:
        raise ValueError("frame header differs from STREAMINFO")
    first = num if variable else num * info["max_blocksize"]
    return dict(bs=bs, first_sample=first, assign=assign, channels=channels, bps=bps, end=p + 1)


FIXED_COEFS = [[], [1], [2, -1], [3, -3, 1], [4, -6, 4, -1]]


def _residual(r, bs, order):
    method = r.u(2)
    if method > 1:
        raise ValueError("reserved residual coding method")
    pbits, esc = (4, 15) if method == 0 else (5, 31)
    po = r.u(4)
    if bs % (1 << po) or (bs >> po) < order:
        raise ValueError("bad partition order")
    out = []
    for p in range(1 << po):
        n = (bs >> po) - (order if p == 0 else 0)
        k = r.u(pbits)
        if k == esc:
            nb = r.u(5)
            out += [r.s(nb) for _ in range(n)]
        else:
            for _ in range(n):
                u = (r.unary() << k) | r.u(k)
                out.append((u >> 1) ^ -(u & 1))
    return out


def _restore(warm, res, coefs, shift):
    s = list(warm)
    o = len(coefs)
    for e in res:
        acc = 0
        for j in range(o):
            acc += coefs[j] * s[-1 - j]
        s.append(e + (acc >> shift))
    return s


def _subframe(r, bs, bps):
    if r.u(1):
        raise ValueError("subframe padding bit set")
    t = r.u(6)
    wasted = 0
    if r.u(1):
        wasted = r.unary() + 1
        if wasted >= bps:
            raise ValueError("wasted bits exceed the sample size")
    b = bps - wasted
    if t == 0:
        s = [r.s(b)] * bs
    elif t == 1:
        s = [r.s(b) for _ in range(bs)]
    elif 8 <= t <= 12:
        o = t - 8
        warm = [r.s(b) for _ in range(o)]
        s = _restore(warm, _residual(r, bs, o), FIXED_COEFS[o], 0)
    elif t >= 32:
        o = t - 31
        warm = [r.s(b) for _ in range(o)]
        prec = r.u(4) + 1
        if prec == 16:
            raise ValueError("reserved LPC precision")
        shift = r.s(5)
        if shift < 0:
            raise ValueError("negative LPC shift")
        coefs = [r.s(prec) for _ in range(o)]
        s = _restore(warm, _residual(r, bs, o), coefs, shift)
    else:
        raise ValueError("reserved subframe type")
    if len(s) != bs:
        raise ValueError("bad subframe length")
    return np.asarray(s, dtype=np.int64) << wasted


def decode_frame(buf, pos, info):
    """-> (header dict, int64 [channels, bs], byte offset after the frame).  Checks the CRC-16."""
    h = parse_header(buf, pos, info)
    r = Bits(buf, h["end"])
    a, bps = h["assign"], h["bps"]
    ch = []
    for c in range(h["channels"]):
        side = (a == 8 and c == 1) or (a == 9 and c == 0) or (a == 10 and c == 1)
        ch.append(_subframe(r, h["bs"], bps + side))
    if a == 8:
        ch[1] = ch[0] - ch[1]
    elif a == 9:
        ch[0] = ch[0] + ch[1]
    elif a == 10:
        mid = (ch[0] << 1) | (ch[1] & 1)
        ch = [(mid + ch[1]) >> 1, (mid - ch[1]) >> 1]
    if r.pos & 7 and r.u(8 - (r.pos & 7)):
        raise ValueError("non-zero frame padding")
    end = (r.pos >> 3) + 2
    if end > len(buf):
        raise ValueError("truncated frame")
    if crc16(buf[pos: end - 2]) != int.from_bytes(buf[end - 2: end], "big"):
        raise ValueError("frame CRC-16 mismatch")
    return h, np.stack(ch), end


def md5_of(pcm, bps):
    """MD5 of the interleaved little-endian samples, ceil(bps / 8) bytes each (what STREAMINFO stores)."""
    nb = (bps + 7) // 8
    x = np.asarray(pcm, dtype=np.int64).T.reshape(-1)
    b = (x & ((1 << (8 * nb)) - 1)).astype("<u8").view(np.uint8).reshape(-1, 8)[:, :nb]
    return hashlib.md5(b.tobytes()).digest()


def decode(buf, check_md5=True):
    """-> (info, int64 [channels, total_samples], list of (frame offset, frame end)).  ValueError on anything malformed."""
    buf = bytes(buf)
    info = parse_streaminfo(buf)
    if info["total_samples"] == 0:
        raise ValueError("unknown total sample count")
    pos, n, blocks, frames = info["first_frame"], 0, [], []
    while n < info["total_samples"]:
        h, x, end = decode_frame(buf, pos, info)
        if h["first_sample"] != n or n + h["bs"] > info["total_samples"]:
            raise ValueError("frame sample number out of sequence")
        blocks.append(x)
        frames.append((pos, end))
        n += h["bs"]
        pos = end
    pcm = np.concatenate(blocks, axis=1)
    if check_md5 and info["md5"] != bytes(16) and md5_of(pcm, info["bps"]) != info["md5"]:
        raise ValueError("MD5 mismatch")
    return info, pcm, frames


def waveform(pcm, bps):
    """float32 [N]: each channel as s / 2^(bps-1) in float32, averaged in channel order, times 2^15 -- what
    get_waveform(normalization=False) returns for the same PCM in a WAVE file."""
    x = np.asarray(pcm, dtype=np.float32) * np.float32(2.0 ** (1 - bps))
    acc = x[0].copy()
    for c in range(1, x.shape[0]):
        acc = acc + x[c]
    if x.shape[0] > 1:
        acc = acc / np.float32(x.shape[0])
    return (acc * np.float32(32768.0)).astype(np.float32)
