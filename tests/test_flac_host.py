"""FLAC on the host: the numpy decoder of oracle/flac.py against real libFLAC output (the LibriSpeech fixture's
STREAMINFO MD5 and frame CRC-16s), the synthetic streams of oracle/flac_encode.py, the STREAMINFO parser of
espresso_b200.data.flac and its refusals, frame counts from STREAMINFO, and FLAC manifests -> packed batches."""
import functools
import io
import os

import numpy as np
import pytest
import torch

from flac_util import corpus

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "librispeech_6313-76958-0021.flac")


@functools.lru_cache(maxsize=1)
def _streams():
    from oracle import flac_encode as E

    return E.synthetic_streams()


def _fixture():
    with open(FIXTURE, "rb") as f:
        return f.read()


def test_oracle_decodes_the_librispeech_fixture_to_its_md5_and_crcs():
    from oracle import flac as F

    buf = _fixture()
    info, pcm, frames = F.decode(buf)  # raises on any CRC-8 / CRC-16 / MD5 mismatch
    assert (info["sample_rate"], info["channels"], info["bps"], info["total_samples"]) == (16000, 1, 16, 190800)
    assert F.md5_of(pcm, 16) == info["md5"] != bytes(16)
    assert len(frames) == 47 and frames[-1][1] == len(buf)
    for a, e in frames:
        assert F.crc16(buf[a: e - 2]) == int.from_bytes(buf[e - 2: e], "big")


def test_synthetic_streams_round_trip_exactly():
    from oracle import flac as F

    names = set()
    for name, buf, pcm, bps in _streams():
        info, got, _ = F.decode(buf)
        assert info["bps"] == bps and info["channels"] == pcm.shape[0] and np.array_equal(got, pcm), name
        assert F.md5_of(pcm, bps) == info["md5"]
        names.add(name)
    assert {"fake_sync", "stereo16_variable", "mono16_block16", "mono24_lpc_orders"} <= names


def test_fake_sync_stream_holds_a_valid_frame_off_the_chain():
    """The VERBATIM samples of frame 1 contain a whole frame (CRC-8 and CRC-16 valid) that claims samples of frame 3."""
    from oracle import flac as F

    buf = dict((n, b) for n, b, _, _ in _streams())["fake_sync"]
    info, _, frames = F.decode(buf)
    a, e = frames[1]
    hits = [p for p in range(a + 1, e) if buf[p] == 0xFF and buf[p + 1] & 0xFE == 0xF8]
    found = []
    for p in hits:
        try:
            h, x, end = F.decode_frame(buf, p, info)
        except ValueError:
            continue
        found.append((p, h["first_sample"], end))
    assert len(found) == 1 and found[0][1] == 3 * info["max_blocksize"] and found[0][2] <= e
    assert all(p != found[0][0] for p, _ in frames)


def test_parser_reports_parameters_and_sample_counts():
    from espresso_b200.data import flac as FL
    from oracle import flac as F

    for name, buf, pcm, bps in list(_streams()) + [("fixture", _fixture(), None, 16)]:
        want = F.parse_streaminfo(buf)
        s = FL.read_stream(buf)
        got = s.info
        assert (got.sample_rate, got.channels, got.bps, got.total_samples, got.md5, got.max_blocksize, got.first_frame) == \
            (want["sample_rate"], want["channels"], want["bps"], want["total_samples"], want["md5"], want["max_blocksize"],
             want["first_frame"]), name
        assert s.frames == buf[got.first_frame:] and s.total_samples == want["total_samples"]
        if pcm is not None:
            assert got.total_samples == pcm.shape[1]


def test_num_frames_of_reads_streaminfo():
    from espresso_b200.data.audio_io import num_frames_of

    want = 1 + (190800 - 400) // 160
    assert num_frames_of(FIXTURE) == want
    fp = io.BytesIO(_fixture())
    assert num_frames_of(fp) == want and fp.tell() == 0


def _patch(buf, bps=None, total=None):
    """Rewrite STREAMINFO's bits-per-sample or total sample count."""
    b = bytearray(buf)
    v = int.from_bytes(b[18:26], "big")
    if bps is not None:
        v = (v & ~(31 << 36)) | ((bps - 1) << 36)
    if total is not None:
        v = (v & ~((1 << 36) - 1)) | total
    b[18:26] = v.to_bytes(8, "big")
    return bytes(b)


def test_parser_refuses_malformed_streams():
    from espresso_b200.data import flac as FL

    buf = dict((n, b) for n, b, _, _ in _streams())["mono16_subframe_types"]
    FL.read_stream(buf)
    bad = {
        "truncated": buf[:30],
        "marker": b"fLaX" + buf[4:],
        "no streaminfo": b"fLaC" + bytes([0x81, 0, 0, 4]) + bytes(4),
        "32-bit": _patch(buf, bps=32),
        "unknown total": _patch(buf, total=0),
        "empty": b"",
    }
    for name, b in bad.items():
        with pytest.raises(ValueError):
            FL.read_stream(b)
        with pytest.raises(ValueError):
            FL.read_info(io.BytesIO(b))


def test_flac_manifest_builds_packed_batches(tmp_path):
    from espresso_b200.data import flac as FL
    from espresso_b200.data.asr_dataset import get_asr_dataset_from_json
    from espresso_b200.data.collate import collate

    d, fdir, wdir, pcms = corpus(tmp_path, n=6)
    spec = "{'freq_mask_F': 10, 'freq_mask_N': 2, 'time_mask_pm': 0.2, 'time_mask_ps': 0.2, 'time_warp_W': 5}"
    dsf = get_asr_dataset_from_json(fdir, "test", d, is_training_set=True, specaugment_config=spec, seed=3)
    dsw = get_asr_dataset_from_json(wdir, "test", d, is_training_set=True, specaugment_config=spec, seed=3)
    # frame counts come from STREAMINFO and equal the WAVE ones, so the SpecAugment draws are the same
    assert dsf.src_sizes.tolist() == dsw.src_sizes.tolist() == [1 + (pcms[u].shape[1] - 400) // 160 for u in dsf.src.utt_ids]
    idx = [0, 3, 4, 1]
    bf = dsf.collater([dsf[i] for i in idx])
    bw = dsw.collater([dsw[i] for i in idx])
    nf, nw = bf["net_input"], bw["net_input"]
    p = nf["src_tokens"]
    assert isinstance(p, FL.PackedFlac) and p.batch == 4 and p.width == nw["src_tokens"].shape[1]
    assert torch.equal(nf["src_lengths"], nw["src_lengths"]) and torch.equal(p.lengths, nw["src_lengths"])
    assert bf["utt_id"] == bw["utt_id"] == p.names
    for k in ("freq_masks", "time_masks", "time_warp", "target", "prev_output_tokens"):
        got, want = (nf.get(k), nw.get(k)) if k != "target" else (bf[k], bw[k])
        assert torch.equal(got, want), k
    params, offsets, frames = p.views(p.buffer)
    assert offsets[0] == 0 and offsets[-1] == frames.numel() and p.buffer.numel() == 8 * (5 * 4 + 5) + frames.numel()
    for b, u in enumerate(bf["utt_id"]):
        raw = open(os.path.join(fdir, u + ".flac"), "rb").read()
        info = FL.read_info(io.BytesIO(raw))
        assert bytes(frames[offsets[b]: offsets[b + 1]].numpy()) == raw[info.first_frame:]
        assert params[b].tolist() == [pcms[u].shape[1], 16000, 1, 16, 4096]
    # one batch is one format; "command" entries whose output is FLAC are FLAC items too
    with pytest.raises(ValueError, match="mixes FLAC"):
        collate([dsf[0], dsw[1]], 1, 2)
    from espresso_b200.data.asr_dataset import AudioFeatDataset

    cmd = AudioFeatDataset(["a"], ["cat %s |" % os.path.join(fdir, "u02.flac")], feat_dim=80, feature_type="fbank")
    assert isinstance(cmd[0]["source"], FL.FlacStream) and cmd.sizes[0] == 1 + (pcms["u02"].shape[1] - 400) // 160
