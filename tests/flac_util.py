"""Test helpers: the same utterances as FLAC files (oracle/flac_encode.py) and as WAVE files, with JSON manifests."""
import json
import os
import struct

import numpy as np


def write_wav(path, pcm, bps, rate=16000):
    """Integer PCM [channels, N] as a RIFF/WAVE file of 8 (unsigned), 16 or 24 bits."""
    x = np.asarray(pcm, dtype=np.int64).T.reshape(-1)
    nb = bps // 8
    if bps == 8:
        data = (x + 128).astype(np.uint8).tobytes()
    else:
        data = (x & ((1 << bps) - 1)).astype("<u4").view(np.uint8).reshape(-1, 4)[:, :nb].tobytes()
    C = pcm.shape[0]
    fmt = struct.pack("<HHIIHH", 1, C, rate, rate * C * nb, C * nb, bps)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", len(data)) + data
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", len(body)) + body)


def librispeech_like(pcm, rate=16000, block=4096):
    """16-bit mono at flac -5-like settings: fixed 4096-sample blocks, LPC order 8, Rice partitions of order 4."""
    from oracle import flac_encode as E

    n = pcm.shape[1]
    sizes = [block] * (n // block) + ([n % block] if n % block else [])
    return E.encode(pcm, 16, rate, [{"bs": s, "subs": [{"kind": "lpc", "order": 8, "precision": 12,
                                                        "part_order": 4 if s % 16 == 0 and s >= 256 else 0}]}
                                    for s in sizes])


def speech_like(rs, n):
    """int16-range noise + tone [1, n], like the synthetic utterances of the other pipeline tests."""
    t = np.arange(n) / 16000.0
    x = 3000.0 * rs.standard_normal(n) + 1500.0 * np.sin(2 * np.pi * rs.uniform(80, 400) * t)
    return np.clip(np.round(x), -32768, 32767).astype(np.int64)[None]


def corpus(tmp_path, n=7, seed=2):
    """-> (dictionary, flac manifest dir, wave manifest dir, {utt: pcm}): test.json in each dir lists the same
    utterances and transcripts, as .flac files in one and .wav files in the other."""
    from espresso_b200.data.asr_dictionary import AsrDictionary

    rs = np.random.RandomState(seed)
    d = AsrDictionary()
    for c in "abcdefghij":
        d.add_symbol(c)
    d.add_symbol("<space>")
    d.space_index = d.index("<space>")
    d.build_bpe("characters_asr")
    fdir, wdir = str(tmp_path / "flac"), str(tmp_path / "wave")
    os.makedirs(fdir, exist_ok=True)
    os.makedirs(wdir, exist_ok=True)
    mf, mw, pcms = {}, {}, {}
    for i in range(n):
        uid = "u%02d" % i
        pcm = speech_like(rs, 5000 + 1700 * ((i * 3) % n))
        text = " ".join("".join(rs.choice(list("abcdefghij"), size=rs.randint(1, 5))) for _ in range(1 + i % 3))
        with open(os.path.join(fdir, uid + ".flac"), "wb") as f:
            f.write(librispeech_like(pcm))
        write_wav(os.path.join(wdir, uid + ".wav"), pcm, 16)
        mf[uid] = {"wave": os.path.join(fdir, uid + ".flac"), "text": text}
        mw[uid] = {"wave": os.path.join(wdir, uid + ".wav"), "text": text}
        pcms[uid] = pcm
    for dd, m in ((fdir, mf), (wdir, mw)):
        with open(os.path.join(dd, "test.json"), "w") as f:
            json.dump(m, f)
    return d, fdir, wdir, pcms
