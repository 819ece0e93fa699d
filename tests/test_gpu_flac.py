"""GPU: esp_flac_decode (csrc/flac.cu) through the C ABI against the numpy decoder of oracle/flac.py, bit for bit: the
LibriSpeech fixture (real libFLAC output, MD5 checked), every synthetic stream of oracle/flac_encode.py in one batch,
the zero tail and the bounds of `out`, the false sync, single-byte corruptions, equality with get_waveform on the same
PCM as WAVE (and so with its filterbank), and a training step and recognize() from a FLAC manifest against a WAVE one."""
import functools
import os

import numpy as np
import pytest
import torch

from flac_util import corpus, write_wav

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "librispeech_6313-76958-0021.flac")


@functools.lru_cache(maxsize=1)
def _streams():
    from oracle import flac_encode as E

    with open(FIXTURE, "rb") as f:
        fixture = f.read()
    return [("fixture", fixture)] + [(n, b) for n, b, _, _ in E.synthetic_streams()]


@functools.lru_cache(maxsize=None)
def _oracle(buf):
    from oracle import flac as F

    info, pcm, _ = F.decode(buf)
    return info, pcm, F.waveform(pcm, info["bps"])


def _decode(bufs, ld=None, check=False):
    from espresso_b200 import ops
    from espresso_b200.data import flac as FL

    p = FL.pack([FL.read_stream(b) for b in bufs])
    t = p.buffer.to(DEV)
    params, offsets, frames = p.views(t)
    out, st = ops.flac_decode(frames, offsets, params, ld or p.width, p.max_channels, check=check)
    return out.cpu().numpy(), st.cpu().numpy()


def test_fixture_decodes_bit_identical_with_its_md5():
    from oracle import flac as F

    buf = _streams()[0][1]
    info, pcm, want = _oracle(buf)
    out, st = _decode([buf])
    assert st.tolist() == [0] and out.shape == (1, 190800)
    assert np.array_equal(out[0], want)
    assert F.md5_of(out[0].astype(np.int64)[None], 16) == info["md5"]  # 16-bit mono: the samples themselves


def test_every_stream_in_one_batch_bit_identical_with_zero_tails():
    bufs = [b for _, b in _streams()]
    ld = max(_oracle(b)[0]["total_samples"] for b in bufs) + 37
    out, st = _decode(bufs, ld=ld)
    assert st.tolist() == [0] * len(bufs)
    for i, (name, b) in enumerate(_streams()):
        info, pcm, want = _oracle(b)
        n = info["total_samples"]
        assert np.array_equal(out[i, :n], want), name
        assert not out[i, n:].any(), name


def test_nothing_outside_the_output_rows_is_written():
    from espresso_b200 import lib
    from espresso_b200.data import flac as FL

    bufs = [b for n, b in _streams() if n in ("fake_sync", "bps8_ch2", "mono16_block16")]
    p = FL.pack([FL.read_stream(b) for b in bufs])
    t = p.buffer.to(DEV)
    params, offsets, frames = p.views(t)
    B, ld, guard = len(bufs), p.width + 5, 4096
    big = torch.full((guard + B * ld + guard,), -7.25, device=DEV)
    status = torch.full((B + 2,), -9, dtype=torch.int32, device=DEV)
    L = lib.load()
    ws = torch.empty(int(L.esp_flac_decode_workspace_bytes(B, frames.numel(), p.max_channels, ld)), dtype=torch.uint8, device=DEV)
    lib.check(L.esp_flac_decode(frames.data_ptr(), frames.numel(), offsets.data_ptr(), params.data_ptr(), B, p.max_channels,
                                big.data_ptr() + 4 * guard, ld, status.data_ptr() + 4, ws.data_ptr(),
                                torch.cuda.current_stream().cuda_stream))
    big, status = big.cpu().numpy(), status.cpu().numpy()
    assert (big[:guard] == -7.25).all() and (big[guard + B * ld:] == -7.25).all()
    assert status[0] == -9 and status[-1] == -9 and status[1:-1].tolist() == [0] * B
    rows = big[guard: guard + B * ld].reshape(B, ld)
    for i, b in enumerate(bufs):
        info, _, want = _oracle(b)
        n = info["total_samples"]
        assert np.array_equal(rows[i, :n], want) and not rows[i, n:].any()


def test_false_sync_inside_verbatim_data_never_reaches_the_output():
    from oracle import flac_encode as E

    buf, pcm = E.fake_sync_stream()
    out, st = _decode([buf])
    assert st.tolist() == [0] and np.array_equal(out[0], pcm[0].astype(np.float32))


def test_single_byte_corruptions_fail_only_their_utterance():
    from espresso_b200 import lib
    from oracle import flac as F

    good = dict(_streams())["mono16_subframe_types"]
    info, _, frames = F.decode(good)
    a, e = frames[3]  # a FIXED order 1 frame
    hdr = bytearray(good)
    hdr[a + 4] ^= 0x01      # frame number byte: CRC-8 fails, no frame where frame 2 ended
    res = bytearray(good)
    res[(a + e) // 2] ^= 0x10  # inside the residual
    crc = bytearray(good)
    crc[e - 1] ^= 0xFF      # the CRC-16 itself
    other = dict(_streams())["stereo16_assignments"]
    bufs = [other, bytes(hdr), good, bytes(res), bytes(crc), other]
    out, st = _decode(bufs)
    assert st[[0, 2, 5]].tolist() == [0, 0, 0]
    assert st[1] == 2 and st[3] != 0 and st[4] == 4
    for i in (0, 2, 5):
        want = _oracle(bufs[i])[2]
        assert np.array_equal(out[i, : len(want)], want) and not out[i, len(want):].any()
    for i in (1, 3, 4):
        assert not out[i].any()
    with pytest.raises(lib.EspressoB200Error, match="utterance 1: status 2"):
        _decode(bufs, check=True)


@pytest.mark.parametrize("bps,channels", [(16, 1), (16, 2), (24, 2), (8, 3)])
def test_device_waveform_equals_get_waveform_of_the_same_wave(tmp_path, bps, channels):
    """The WAVE path (get_waveform, normalization=False) on the same PCM, bit for bit; hence the same filterbank."""
    from espresso_b200 import ops
    from espresso_b200.data.audio_io import get_waveform
    from oracle import flac_encode as E

    rs = np.random.RandomState(bps + channels)
    pcm = E.synth(rs, channels, 9000, bps)
    buf = E.encode(pcm, bps, 16000, [{"bs": 4096, "assign": 10 if channels == 2 else channels - 1,
                                      "subs": [{"kind": "lpc", "order": 8}]}] * 2 +
                   [{"bs": 808, "assign": 9 if channels == 2 else channels - 1, "subs": [{"kind": "fixed", "order": 2}]}])
    write_wav(str(tmp_path / "x.wav"), pcm, bps)
    want, _ = get_waveform(str(tmp_path / "x.wav"), normalization=False, always_2d=False)
    out, st = _decode([buf])
    assert st.tolist() == [0] and np.array_equal(out[0], want)
    n = torch.tensor([len(want)], dtype=torch.int32, device=DEV)
    fa, _ = ops.frontend_fbank(torch.from_numpy(out).to(DEV), n, out_dtype=torch.float32)
    fb, _ = ops.frontend_fbank(torch.from_numpy(want)[None].to(DEV), n, out_dtype=torch.float32)
    assert torch.equal(fa, fb)


def test_cmvn_tool_reads_flac_like_wave(tmp_path):
    from espresso_b200.tools import compute_global_cmvn_stats as G

    d, fdir, wdir, pcms = corpus(tmp_path, n=4)
    for dd, ext in ((fdir, "flac"), (wdir, "wav")):
        with open(os.path.join(dd, "wav.scp"), "w") as f:
            f.writelines("%s %s\n" % (u, os.path.join(dd, "%s.%s" % (u, ext))) for u in pcms)
        G.main([os.path.join(dd, "wav.scp"), os.path.join(dd, "out"), "--batch-seconds", "0.5"])
    a, b = np.load(os.path.join(fdir, "out", "gcmvn.npz")), np.load(os.path.join(wdir, "out", "gcmvn.npz"))
    assert np.array_equal(a["mean"], b["mean"]) and np.array_equal(a["std"], b["std"])


def test_training_step_and_recognize_from_flac_equal_wave(tmp_path):
    from argparse import Namespace

    from espresso_b200.criterions import CtcLossCriterion
    from espresso_b200.data import flac as FL
    from espresso_b200.data.asr_dataset import get_asr_dataset_from_json
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel, SpeechTransformerModelBase
    from espresso_b200.speech_recognize import recognize
    from espresso_b200.tasks.speech_recognition import SpeechRecognitionEspressoConfig, SpeechRecognitionEspressoTask

    d, fdir, wdir, pcms = corpus(tmp_path, n=7)
    # one training step (CTC, on-the-fly fbank + SpecAugment with time warping) from each manifest
    spec = "{'freq_mask_F': 10, 'freq_mask_N': 2, 'time_mask_pm': 0.1, 'time_mask_ps': 0.1, 'time_warp_W': 5}"

    class _T:
        feat_dim, feat_in_channels, target_dictionary = 80, 1, d

    cfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, layernorm_embedding=True,
        encoder=dict(embed_dim=128, ffn_embed_dim=256, layers=2, attention_heads=2, normalize_before=True, learned_pos=False,
                     relative_positional_embeddings=True, layer_type="conformer", depthwise_conv_kernel_size=15)))
    losses, grads = [], []
    for dd in (fdir, wdir):
        ds = get_asr_dataset_from_json(dd, "test", d, is_training_set=True, specaugment_config=spec, seed=3)
        batch = ds.collater([ds[i] for i in (0, 2, 5, 6)])
        ni = dict(batch["net_input"])
        if isinstance(ni["src_tokens"], FL.PackedFlac):
            ni["src_tokens"], ni["src_lengths"] = FL.to_device(ni["src_tokens"], DEV)
        ni = {k: v.to(DEV) if torch.is_tensor(v) else v for k, v in ni.items() if k != "prev_output_tokens"}
        ni["src_lengths_cpu"] = batch["net_input"]["src_lengths"].long()
        torch.manual_seed(1)
        m = SpeechTransformerEncoderModel.build_model(cfg, _T()).finalize_(DEV)
        m.frontend = OnTheFlyFbank(np.full(80, 15.0), np.full(80, 4.0))
        m.train()
        m.flat.zero_grad()
        loss, _, _ = CtcLossCriterion(_T(), zero_infinity=True, sentence_avg=True)(m, {"net_input": ni, "target": batch["target"].to(DEV)})
        loss.backward()
        torch.cuda.synchronize()
        losses.append(loss.item())
        grads.append(m.flat.grad("encoder.layers.1.self_attn.q_proj.weight").float().cpu())
    assert losses[0] == losses[1] and np.isfinite(losses[0])
    assert torch.equal(grads[0], grads[1])
    # recognize() over each manifest: identical hypotheses and scores
    torch.manual_seed(3)
    mcfg = SpeechTransformerConfig.from_dict(dict(
        dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, layernorm_embedding=False, max_target_positions=64,
        encoder=dict(embed_dim=64, ffn_embed_dim=128, layers=1, attention_heads=4, normalize_before=True, learned_pos=False,
                     relative_positional_embeddings=True, layer_type="transformer"),
        decoder=dict(embed_dim=64, ffn_embed_dim=128, layers=1, attention_heads=4, normalize_before=True, learned_pos=False,
                     relative_positional_embeddings=False, input_dim=64, output_dim=64)))
    lines = []
    model = None
    for dd in (fdir, wdir):
        task = SpeechRecognitionEspressoTask(SpeechRecognitionEspressoConfig(
            criterion_name="label_smoothed_cross_entropy_v2", data=dd, autoregressive=True), d, feat_dim=80)
        if model is None:
            model = SpeechTransformerModelBase.build_model(mcfg, task).finalize_(DEV)
            model.frontend = OnTheFlyFbank(None, None)
        out = recognize(task, [model], subset="test", gen_args=Namespace(beam=2, max_len_a=0.0, max_len_b=6, lm_weight=0.0),
                        max_tokens=None, max_sentences=3, device=DEV)
        assert out["num_sentences"] == len(pcms)
        lines.append(out["lines"])
    assert lines[0] == lines[1]


def test_one_decode_counts_four_launches():
    from espresso_b200 import lib

    bufs = [b for n, b in _streams() if n in ("fixture", "stereo16_variable")]
    _decode(bufs)
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    _decode(bufs)
    assert lib.launch_count() - n0 == 4  # scan, measure, chain, decode
