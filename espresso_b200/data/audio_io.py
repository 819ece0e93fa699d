"""Audio / feature wire formats of the ASR input pipeline (host side; SURVEY.md section 8 row A1 and (f)3).

* `get_waveform` -- fairseq/data/audio/audio_utils.py:69-126: decode an audio file to float32 [channels, samples], mono by
  averaging, scaled to the int16 range when `normalization=False` (what the Kaldi-compatible fbank expects,
  espresso/data/feat_text_dataset.py:137-150).  The reference goes through libsndfile; RIFF/WAVE (PCM 8/16/24/32 bit, IEEE
  float 32/64, WAVE_FORMAT_EXTENSIBLE) is decoded here with numpy alone, other containers (FLAC, OGG) through `soundfile` if
  it is installed.  The training and decoding pipelines do not come here for FLAC: they decode it on the device
  (espresso_b200/data/flac.py), and `num_frames_of` reads a FLAC file's STREAMINFO.
* `read_kaldi_mat` -- the `kaldi_io.read_mat("file.ark:offset")` call of feat_text_dataset.py:69-75,129-130: binary Kaldi
  matrices, float ("FM "), double ("DM ") and the three compressed layouts ("CM ", "CM2", "CM3") of kaldi/src/matrix/
  compressed-matrix.h.  `write_kaldi_mat` writes FM/DM archives + scp lines (tools and tests)."""
import io
import os
import struct

import numpy as np

SF_AUDIO_FILE_EXTENSIONS = {".wav", ".flac", ".ogg"}  # audio_utils.py:20


def _decode_wav(buf):
    if len(buf) < 12 or buf[:4] not in (b"RIFF", b"RF64") or buf[8:12] != b"WAVE":
        raise ValueError("not a RIFF/WAVE stream")
    pos, fmt, data = 12, None, None
    while pos + 8 <= len(buf):
        cid, size = buf[pos: pos + 4], struct.unpack_from("<I", buf, pos + 4)[0]
        body = pos + 8
        if cid == b"fmt ":
            tag, ch, rate, _, _, bits = struct.unpack_from("<HHIIHH", buf, body)
            if tag == 0xFFFE and size >= 26:  # WAVE_FORMAT_EXTENSIBLE: the real tag is the first word of the sub-format GUID
                tag = struct.unpack_from("<H", buf, body + 24)[0]
            fmt = (tag, ch, rate, bits)
        elif cid == b"data":
            if size == 0xFFFFFFFF or body + size > len(buf):  # streamed output (e.g. sph2pipe): data runs to the end
                size = len(buf) - body
            data = buf[body: body + size]
            break
        pos = body + size + (size & 1)
    if fmt is None or data is None:
        raise ValueError("WAVE stream without fmt/data chunk")
    tag, ch, rate, bits = fmt
    if tag == 1:  # integer PCM -> [-1, 1) like libsndfile's float read
        if bits == 8:
            x = (np.frombuffer(data, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
        elif bits == 16:
            x = np.frombuffer(data, dtype="<i2").astype(np.float32) / 32768.0
        elif bits == 24:
            b = np.frombuffer(data[: len(data) // 3 * 3], dtype=np.uint8).reshape(-1, 3).astype(np.int32)
            v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
            x = (v - ((v & 0x800000) << 1)).astype(np.float32) / 8388608.0
        elif bits == 32:
            x = (np.frombuffer(data, dtype="<i4").astype(np.float64) / 2147483648.0).astype(np.float32)
        else:
            raise ValueError("unsupported PCM width: %d bits" % bits)
    elif tag == 3:
        x = np.frombuffer(data, dtype="<f4" if bits == 32 else "<f8").astype(np.float32)
    else:
        raise ValueError("unsupported WAVE format tag %d (PCM and IEEE float only)" % tag)
    n = len(x) // ch
    return x[: n * ch].reshape(n, ch).T, rate


def get_waveform(path_or_fp, normalization=True, mono=True, frames=-1, start=0, always_2d=True, output_sample_rate=None):
    """-> (float32 [channels, samples] or [samples], sample_rate)."""
    if isinstance(path_or_fp, (str, os.PathLike)):
        ext = os.path.splitext(str(path_or_fp))[1].lower()
        if ext not in SF_AUDIO_FILE_EXTENSIONS:
            raise ValueError("Unsupported audio format: %s" % ext)
        with open(path_or_fp, "rb") as f:
            buf = f.read()
    else:
        buf = path_or_fp.read()
    if buf[:4] in (b"RIFF", b"RF64"):
        wav, rate = _decode_wav(buf)
    else:
        try:
            import soundfile as sf
        except ImportError:
            raise ImportError("only RIFF/WAVE is decoded natively; install soundfile for FLAC / OGG input")
        wav, rate = sf.read(io.BytesIO(buf), dtype="float32", always_2d=True)
        wav = wav.T
    if start < 0:
        start += wav.shape[1]
    wav = wav[:, start: (None if frames < 0 else start + frames)]
    if mono and wav.shape[0] > 1:
        wav = wav.mean(axis=0, keepdims=True)
    if output_sample_rate is not None and output_sample_rate != rate:
        raise NotImplementedError("resampling (sox effects in the reference) is not on the path: prepare %d Hz audio" % output_sample_rate)
    wav = np.ascontiguousarray(wav, dtype=np.float32)
    if not normalization:
        wav = wav * 2 ** 15  # audio_utils.py:117-118
    return (wav if always_2d else wav.squeeze(0)), rate


# ---- Kaldi matrices ---------------------------------------------------------------------------------------------------
def _read_token(f):
    tok = b""
    while True:
        c = f.read(1)
        if not c or c == b" ":
            return tok
        tok += c


def _read_i32(f):
    assert f.read(1) == b"\x04"
    return struct.unpack("<i", f.read(4))[0]


def _uncompress(f, fmt):
    gmin, grange, rows, cols = struct.unpack("<ffii", f.read(16))
    if fmt == b"CM":  # per-column headers (4 x uint16 percentiles) + uint8 data, column-major
        hdr = np.frombuffer(f.read(cols * 8), dtype="<u2").reshape(cols, 4).astype(np.float32)
        p = gmin + grange * (1.0 / 65535.0) * hdr                         # p0, p25, p75, p100 per column
        d = np.frombuffer(f.read(rows * cols), dtype=np.uint8).reshape(cols, rows).astype(np.float32)
        p0, p25, p75, p100 = (p[:, i: i + 1] for i in range(4))
        out = np.where(d <= 64, p0 + (p25 - p0) * d * (1 / 64.0),
                       np.where(d <= 192, p25 + (p75 - p25) * (d - 64) * (1 / 128.0), p75 + (p100 - p75) * (d - 192) * (1 / 63.0)))
        return out.T.astype(np.float32)
    if fmt == b"CM2":
        d = np.frombuffer(f.read(rows * cols * 2), dtype="<u2").reshape(rows, cols).astype(np.float32)
        return (gmin + grange * (1.0 / 65535.0) * d).astype(np.float32)
    d = np.frombuffer(f.read(rows * cols), dtype=np.uint8).reshape(rows, cols).astype(np.float32)  # CM3
    return (gmin + grange * (1.0 / 255.0) * d).astype(np.float32)


def read_kaldi_mat(rxfile):
    """"path/to/feats.ark:12345" (or an open binary stream positioned at the matrix) -> float32 [frames, dim]."""
    if isinstance(rxfile, str):
        path, _, off = rxfile.strip().rpartition(":")
        if not path or not off.isdigit():
            raise ValueError("expected 'file.ark:offset', got %r" % rxfile)
        with open(path, "rb") as f:
            f.seek(int(off))
            return read_kaldi_mat(f)
    f = rxfile
    if f.read(2) != b"\x00B":
        raise ValueError("only binary Kaldi matrices are supported")
    fmt = _read_token(f)
    if fmt in (b"CM", b"CM2", b"CM3"):
        return _uncompress(f, fmt)
    if fmt not in (b"FM", b"DM"):
        raise ValueError("unknown Kaldi matrix type %r" % fmt)
    rows, cols = _read_i32(f), _read_i32(f)
    dt = "<f4" if fmt == b"FM" else "<f8"
    return np.frombuffer(f.read(rows * cols * int(dt[-1])), dtype=dt).reshape(rows, cols).astype(np.float32)


def write_kaldi_mat(f, key, mat):
    """Append one binary matrix to an open ark stream; returns the byte offset an scp line should point to."""
    mat = np.ascontiguousarray(mat)
    f.write(key.encode() + b" ")
    off = f.tell()
    tag = b"FM " if mat.dtype == np.float32 else b"DM "
    if mat.dtype not in (np.float32, np.float64):
        raise ValueError("float32 / float64 matrices only")
    f.write(b"\x00B" + tag + b"\x04" + struct.pack("<i", mat.shape[0]) + b"\x04" + struct.pack("<i", mat.shape[1]))
    f.write(mat.astype("<f4" if mat.dtype == np.float32 else "<f8").tobytes())
    return off


def num_frames_of(rxfile, frame_length_ms=25.0, frame_shift_ms=10.0):
    """espresso/tools/utils.py compute_num_frames_from_feat_or_waveform: rows of a Kaldi matrix, or the snip-edges frame
    count of a waveform file (1 + (samples - window) // shift)."""
    if isinstance(rxfile, str) and rxfile.strip().rpartition(":")[2].isdigit() and ".ark:" in rxfile:
        return int(read_kaldi_mat(rxfile).shape[0])
    info = _flac_info(rxfile)
    if info is not None:  # FLAC: the sample count is in STREAMINFO, nothing is decoded
        n, rate = info.total_samples, info.sample_rate
    else:
        wav, rate = get_waveform(rxfile, normalization=False)
        n = wav.shape[1]
    win, hop = int(rate * frame_length_ms / 1000.0), int(rate * frame_shift_ms / 1000.0)
    return max(0, 1 + (n - win) // hop)


def _flac_info(rxfile):
    """STREAMINFO of a .flac path or of a seekable file object that starts with fLaC (left at its start), else None."""
    from .flac import read_info

    if isinstance(rxfile, (str, os.PathLike)):
        if not str(rxfile).lower().endswith(".flac"):
            return None
        with open(rxfile, "rb") as f:
            return read_info(f)
    pos = rxfile.tell()
    head = rxfile.read(4)
    rxfile.seek(pos)
    if head != b"fLaC":
        return None
    info = read_info(rxfile)
    rxfile.seek(pos)
    return info
