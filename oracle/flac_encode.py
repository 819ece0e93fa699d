"""Test-only FLAC encoder (RFC 9639): writes streams whose every frame and subframe is chosen explicitly, so that the
decoders can be tested on each feature of the format, with a correct STREAMINFO MD5, header CRC-8 and frame CRC-16.

    buf = encode(pcm, bps, rate, frames)      # pcm: int [channels, N]; frames: list of FrameSpec
    synthetic_streams()                       # -> [(name, bytes, pcm, bps)]: the set the tests decode

A FrameSpec is a dict: bs (block size), assign (channel assignment 0-10; default independent), subs (one dict per
subframe: kind = constant | verbatim | fixed | lpc, order, precision, rice2, part_order, escape = partition indices,
wasted = True to shift out common trailing zero bits).  It compresses nothing on purpose: it only has to be valid."""
import numpy as np

from .flac import FIXED_COEFS, crc8, crc16, md5_of


class BitWriter:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, n):
        if n == 0:
            return
        self.acc = (self.acc << n) | (int(v) & ((1 << n) - 1))
        self.n += n
        while self.n >= 8:
            self.n -= 8
            self.out.append((self.acc >> self.n) & 0xFF)
        self.acc &= (1 << self.n) - 1

    def unary(self, q):
        for _ in range(q // 32):
            self.put(0, 32)
        self.put(1, q % 32 + 1)

    def align(self):
        if self.n:
            self.put(0, 8 - self.n)

    def bytes(self):
        assert self.n == 0
        return bytes(self.out)


def _utf8(v):
    if v < 0x80:
        return bytes([v])
    n = 2
    while v >= 1 << (5 * n + 1):
        n += 1
    out = []
    for _ in range(n - 1):
        out.append(0x80 | (v & 0x3F))
        v >>= 6
    lead = (0xFF << (8 - n)) & 0xFF
    return bytes([lead | v] + out[::-1])


_BS_CODE = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, **{256 << k: 8 + k for k in range(8)}}
_SR_CODE = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}
_BPS_CODE = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6}


def frame_header(bs, number, variable, assign, bps, rate):
    """Header bytes incl. CRC-8.  `number` is the frame number (fixed blocking) or first sample (variable)."""
    extra_bs = b""
    if bs in _BS_CODE:
        bsc = _BS_CODE[bs]
    elif bs <= 256:
        bsc, extra_bs = 6, bytes([bs - 1])
    else:
        bsc, extra_bs = 7, (bs - 1).to_bytes(2, "big")
    extra_sr = b""
    if rate in _SR_CODE:
        src = _SR_CODE[rate]
    elif rate % 1000 == 0 and rate // 1000 < 256:
        src, extra_sr = 12, bytes([rate // 1000])
    elif rate < 65536:
        src, extra_sr = 13, rate.to_bytes(2, "big")
    elif rate % 10 == 0 and rate // 10 < 65536:
        src, extra_sr = 14, (rate // 10).to_bytes(2, "big")
    else:
        src = 0
    h = bytes([0xFF, 0xF8 | variable, (bsc << 4) | src, (assign << 4) | (_BPS_CODE.get(bps, 0) << 1)])
    h += _utf8(number) + extra_bs + extra_sr
    return h + bytes([crc8(h)])


def _fold(r):
    r = np.asarray(r, dtype=np.int64)
    return np.where(r >= 0, 2 * r, -2 * r - 1)


def _residual(w, res, bs, order, spec):
    rice2, po = spec.get("rice2", False), spec.get("part_order", 0)
    pbits, esc = (5, 31) if rice2 else (4, 15)
    w.put(1 if rice2 else 0, 2)
    w.put(po, 4)
    res = np.asarray(res, dtype=np.int64)
    at = 0
    for p in range(1 << po):
        n = (bs >> po) - (order if p == 0 else 0)
        part = res[at: at + n]
        at += n
        u = _fold(part)
        k = None
        if p not in spec.get("escape", ()):
            best = None
            for kk in range(esc):
                bits = int((u >> kk).sum()) + n * (kk + 1)
                if best is None or bits < best:
                    best, k = bits, kk
        if k is None or (n and int(u.max() >> k) > 4096):
            nb = 0 if not n or not part.any() else int(max(int(part.max()).bit_length(), int((-part.min() - 1)).bit_length())) + 1
            w.put(esc, pbits)
            w.put(nb, 5)
            for v in part:
                w.put(v, nb)
        else:
            w.put(k, pbits)
            for v in u:
                w.unary(int(v) >> k)
                w.put(int(v), k)
    assert at == len(res)


def _lpc_coefs(x, order, precision):
    """Quantised coefficients from an autocorrelation fit (Levinson-Durbin), and their shift."""
    x = np.asarray(x, dtype=np.float64)
    ac = np.array([np.dot(x[: len(x) - k], x[k:]) for k in range(order + 1)]) + 1e-9
    ac[0] *= 1.0 + 1e-9
    a, err = np.zeros(order), ac[0]
    for i in range(order):
        k = (ac[i + 1] - np.dot(a[:i], ac[i:0:-1])) / err
        a[:i] = a[:i] - k * a[:i][::-1]
        a[i] = k
        err *= 1.0 - k * k
    cmax = max(np.abs(a).max(), 1e-9)
    shift = int(np.clip(precision - 1 - (int(np.floor(np.log2(cmax))) + 1), 0, 15))
    q = np.clip(np.round(a * (1 << shift)), -(1 << (precision - 1)), (1 << (precision - 1)) - 1).astype(np.int64)
    return [int(c) for c in q], shift


def _predict(s, coefs, shift):
    s = [int(v) for v in s]
    o = len(coefs)
    return [s[n] - (sum(coefs[j] * s[n - 1 - j] for j in range(o)) >> shift) for n in range(o, len(s))]


def subframe(w, x, bps, spec):
    x = np.asarray(x, dtype=np.int64)
    wasted = 0
    if spec.get("wasted") and x.any():
        while wasted < bps - 1 and not (x & ((2 << wasted) - 1)).any():
            wasted += 1
    x = x >> wasted
    b = bps - wasted
    kind, o = spec["kind"], spec.get("order", 0)
    w.put(0, 1)
    w.put({"constant": 0, "verbatim": 1, "fixed": 8 + o, "lpc": 31 + o}[kind], 6)
    w.put(1 if wasted else 0, 1)
    if wasted:
        w.unary(wasted - 1)
    if kind == "constant":
        assert (x == x[0]).all()
        w.put(x[0], b)
        return
    if kind == "verbatim":
        for v in x:
            w.put(v, b)
        return
    for v in x[:o]:
        w.put(v, b)
    if kind == "fixed":
        res = _predict(x, FIXED_COEFS[o], 0)
    else:
        prec = spec.get("precision", 12)
        coefs, shift = spec["coefs"] if "coefs" in spec else _lpc_coefs(x, o, prec)
        w.put(prec - 1, 4)
        w.put(shift, 5)
        for c in coefs:
            assert -(1 << (prec - 1)) <= c < (1 << (prec - 1))
            w.put(c, prec)
        res = _predict(x, coefs, shift)
    _residual(w, res, len(x), o, spec)


def encode_frame(pcm_block, number, variable, bps, rate, spec):
    """One frame: header, subframes (decorrelated per spec['assign']), padding, CRC-16."""
    x = np.asarray(pcm_block, dtype=np.int64)
    C, bs = x.shape
    a = spec.get("assign", C - 1)
    if a == 8:
        chans, sbps = [x[0], x[0] - x[1]], [bps, bps + 1]
    elif a == 9:
        chans, sbps = [x[0] - x[1], x[1]], [bps + 1, bps]
    elif a == 10:
        chans, sbps = [(x[0] + x[1]) >> 1, x[0] - x[1]], [bps, bps + 1]
    else:
        assert a == C - 1
        chans, sbps = list(x), [bps] * C
    w = BitWriter()
    for b in frame_header(bs, number, variable, a, bps, rate):
        w.put(b, 8)
    subs = spec.get("subs", [{"kind": "fixed", "order": 2}])
    for c in range(C):
        subframe(w, chans[c], sbps[c], subs[c % len(subs)])
    w.align()
    body = w.bytes()
    return body + crc16(body).to_bytes(2, "big")


def streaminfo(min_bs, max_bs, rate, channels, bps, total, md5):
    w = BitWriter()
    w.put(min_bs, 16)
    w.put(max_bs, 16)
    w.put(0, 24)
    w.put(0, 24)
    w.put(rate, 20)
    w.put(channels - 1, 3)
    w.put(bps - 1, 5)
    w.put(total >> 4, 32)  # 36 bits in two pieces
    w.put(total & 15, 4)
    return w.bytes() + md5


def metadata(info_body, extra=True):
    """fLaC + STREAMINFO, then (extra) a VORBIS_COMMENT-typed and a PADDING block the parser must skip."""
    blocks = [(0, info_body)]
    if extra:
        blocks += [(4, b"\x07\x00\x00\x00oracle1\x00\x00\x00\x00"), (1, bytes(37))]
    out = b"fLaC"
    for i, (t, body) in enumerate(blocks):
        out += bytes([(0x80 if i == len(blocks) - 1 else 0) | t]) + len(body).to_bytes(3, "big") + body
    return out


def encode(pcm, bps, rate, frames, variable=False, extra_metadata=True):
    """pcm int [channels, N]; frames: FrameSpecs whose bs sum to N."""
    pcm = np.asarray(pcm, dtype=np.int64)
    C, N = pcm.shape
    sizes = [f["bs"] for f in frames]
    assert sum(sizes) == N
    max_bs = max(sizes)
    if not variable:  # fixed blocking: every frame but the last has the nominal size
        assert all(s == sizes[0] for s in sizes[:-1]) and sizes[-1] <= sizes[0]
        max_bs = sizes[0]
    min_bs = min(sizes[:-1]) if len(sizes) > 1 else sizes[0]
    body, at = b"", 0
    for i, f in enumerate(frames):
        body += encode_frame(pcm[:, at: at + f["bs"]], at if variable else i, int(variable), bps, rate, f)
        at += f["bs"]
    return metadata(streaminfo(min_bs, max_bs, rate, C, bps, N, md5_of(pcm, bps)), extra_metadata) + body


def synth(rs, channels, n, bps, wasted=0):
    """Tones + noise filling a good part of the bps range, as ints (low `wasted` bits zero)."""
    t = np.arange(n)
    amp = 0.4 * (1 << (bps - 1))
    out = []
    for c in range(channels):
        f = rs.uniform(0.002, 0.05, size=3)
        x = amp * (0.5 * np.sin(2 * np.pi * f[0] * t) + 0.3 * np.sin(2 * np.pi * f[1] * t + c) + 0.1 * np.sin(2 * np.pi * f[2] * t))
        x = x + rs.standard_normal(n) * amp * 0.02
        x = np.clip(np.round(x), -(1 << (bps - 1)), (1 << (bps - 1)) - 1).astype(np.int64)
        out.append((x >> wasted) << wasted)
    return np.stack(out)


def fake_sync_stream():
    """16-bit mono, fixed blocks of 256: frame 1 is VERBATIM, and its samples hold a COMPLETE valid frame (header with a
    good CRC-8, a CONSTANT subframe, a good CRC-16) claiming to be frame 3.  Only the chain of frames starting at the
    first frame may reach the output."""
    rs = np.random.RandomState(11)
    bps, rate, bs = 16, 16000, 256
    pcm = synth(rs, 1, 4 * bs, bps)
    fake = bytearray(frame_header(16, 3, 0, 0, bps, rate))
    w = BitWriter()
    w.put(0, 8)           # CONSTANT subframe, no wasted bits
    w.put(-12345, 16)
    fake += w.bytes()
    fake += crc16(bytes(fake)).to_bytes(2, "big")
    if len(fake) % 2:
        fake += b"\x00"
    words = np.frombuffer(bytes(fake), dtype=">i2").astype(np.int64)
    pcm[0, bs + 10: bs + 10 + len(words)] = words
    frames = [{"bs": bs, "subs": [{"kind": "fixed", "order": 2}]}, {"bs": bs, "subs": [{"kind": "verbatim"}]},
              {"bs": bs, "subs": [{"kind": "lpc", "order": 4}]}, {"bs": bs, "subs": [{"kind": "fixed", "order": 1}]}]
    return encode(pcm, bps, rate, frames), pcm


def synthetic_streams():
    """[(name, bytes, pcm, bps)] covering every subframe type, stereo mode, LPC order 1-32 with several precisions and
    shifts, wasted bits, Rice2 and escaped partitions, partition orders 0-15, bit depths 4-24, 1-8 channels, fixed and
    variable blocking, a short last block, a block size of 16 and of 65535, and a false sync inside VERBATIM data."""
    rs = np.random.RandomState(2024)
    out = []

    # 16-bit mono: every subframe type and FIXED order, a constant block, a short last block
    pcm = synth(rs, 1, 7 * 1152 + 500, 16)
    pcm[0, 1152: 2304] = 321
    kinds = [{"kind": "fixed", "order": 2}, {"kind": "constant"}, {"kind": "verbatim"}] + \
            [{"kind": "fixed", "order": o, "part_order": o} for o in range(5)]
    out.append(("mono16_subframe_types", encode(pcm, 16, 16000, [{"bs": 1152, "subs": [k]} for k in kinds[:7]] +
                                                [{"bs": 500, "subs": [{"kind": "fixed", "order": 4, "part_order": 2}]}]), pcm, 16))

    # 16-bit stereo: the four channel assignments, FIXED and LPC, Rice2 in some
    pcm = synth(rs, 2, 8 * 576, 16)
    frames = []
    for i in range(8):
        sub = {"kind": "lpc", "order": 8, "precision": 12, "rice2": bool(i & 1)} if i % 3 else {"kind": "fixed", "order": 3}
        frames.append({"bs": 576, "assign": [1, 8, 9, 10][i % 4], "subs": [sub]})
    out.append(("stereo16_assignments", encode(pcm, 16, 44100, frames), pcm, 16))

    # 24-bit mono: LPC orders 1-32, precisions 2-15 (shift follows the coefficients), wasted bits in some
    pcm = synth(rs, 1, 32 * 256, 24)
    frames = [{"bs": 256, "subs": [{"kind": "lpc", "order": o, "precision": 2 + (o * 5) % 14, "part_order": o % 3}]}
              for o in range(1, 33)]
    out.append(("mono24_lpc_orders", encode(pcm, 24, 48000, frames), pcm, 24))

    # explicit shifts 0 and 15 with hand-picked coefficients (LPC restatement of FIXED order 2 and a scaled one)
    pcm = synth(rs, 1, 3 * 1024, 16)
    frames = [{"bs": 1024, "subs": [{"kind": "lpc", "order": 2, "precision": 4, "coefs": ([2, -1], 0)}]},
              {"bs": 1024, "subs": [{"kind": "lpc", "order": 2, "precision": 15, "coefs": ([16383, -8000], 15)}]},
              {"bs": 1024, "subs": [{"kind": "lpc", "order": 3, "precision": 9, "coefs": ([200, -100, 10], 7)}]}]
    out.append(("mono16_lpc_shifts", encode(pcm, 16, 16000, frames), pcm, 16))

    # wasted bits: 24-bit stereo whose low 5 bits are zero, mid/side and independent; a 20-bit one with 3 wasted bits
    pcm = synth(rs, 2, 4 * 1024, 24, wasted=5)
    frames = [{"bs": 1024, "assign": a, "subs": [{"kind": k, "order": 2, "wasted": True}]}
              for a, k in ((10, "lpc"), (1, "fixed"), (8, "verbatim"), (9, "lpc"))]
    out.append(("stereo24_wasted_bits", encode(pcm, 24, 96000, frames), pcm, 24))
    pcm = synth(rs, 1, 2 * 2304, 20, wasted=3)
    frames = [{"bs": 2304, "subs": [{"kind": "fixed", "order": 2, "wasted": True}]},
              {"bs": 2304, "subs": [{"kind": "lpc", "order": 10, "wasted": True}]}]
    out.append(("mono20_wasted_bits", encode(pcm, 20, 22050, frames), pcm, 20))

    # Rice2, escaped partitions (incl. a 0-bit one) and partition orders 0-15; block sizes 32768 and 65535
    pcm = synth(rs, 1, 4 * 4096 + 32768 + 65535, 16)
    pcm[0, 4096: 4096 + 256] = 0
    frames = [{"bs": 4096, "subs": [{"kind": "fixed", "order": 1, "rice2": True, "part_order": 4}]},
              {"bs": 4096, "subs": [{"kind": "fixed", "order": 0, "part_order": 4, "escape": (0, 1, 5)}]},
              {"bs": 4096, "subs": [{"kind": "lpc", "order": 12, "part_order": 8, "rice2": True, "escape": (3,)}]},
              {"bs": 4096, "subs": [{"kind": "fixed", "order": 4, "part_order": 10}]},
              {"bs": 32768, "subs": [{"kind": "fixed", "order": 1, "part_order": 15, "rice2": True}]},
              {"bs": 65535, "subs": [{"kind": "lpc", "order": 32, "precision": 15}]}]
    out.append(("mono16_partitions", encode(pcm, 16, 16000, frames, variable=True), pcm, 16))

    # bit depths 4, 8 and 12 (4 only through STREAMINFO), 8 channels, 3 channels at 20 bits
    for bps, C, rate in ((4, 1, 8000), (8, 2, 8000), (12, 1, 12345), (20, 3, 37000), (16, 8, 32000)):
        pcm = synth(rs, C, 3 * 1000 + 77, bps)
        frames = [{"bs": 1000, "subs": [{"kind": "lpc", "order": 6}, {"kind": "fixed", "order": 2}]}] * 3
        frames.append({"bs": 77, "subs": [{"kind": "verbatim"}]})
        out.append(("bps%d_ch%d" % (bps, C), encode(pcm, bps, rate, frames), pcm, bps))

    # variable blocking with odd sizes (sample numbers coded in 1-3 bytes), and fixed blocks of 16 (2-byte frame numbers)
    sizes = [1000, 16, 4097, 333, 19, 60000, 1]
    pcm = synth(rs, 2, sum(sizes), 16)
    out.append(("stereo16_variable", encode(pcm, 16, 16000, [{"bs": s, "assign": 8, "subs": [{"kind": "fixed" if s > 2 else "verbatim", "order": 2}]}
                                                              for s in sizes], variable=True), pcm, 16))
    pcm = synth(rs, 1, 300 * 16 + 9, 16)
    out.append(("mono16_block16", encode(pcm, 16, 16000, [{"bs": 16, "subs": [{"kind": "fixed", "order": 1}]}] * 300 +
                                         [{"bs": 9, "subs": [{"kind": "verbatim"}]}], extra_metadata=False), pcm, 16))

    buf, pcm = fake_sync_stream()
    out.append(("fake_sync", buf, pcm, 16))
    return out
