"""CTC decoding cost on the benchmarked Conformer-CTC (17 x 512, V = 5004, random initialisation): bsz 24 x 10 s utterances
(the recipe's decode batching), greedy vs prefix beam search at beam 10 and 60, with and without the recipe-sized LSTM LM
(lstm_lm_librispeech.yaml: 4 x 800, shared embedding).  Prints one JSON line:
  encoder / search milliseconds per batch (CUDA events; the search includes the final device-to-host copy), RTF,
  per-kernel times of esp_ctc_beam_frames / esp_ctc_beam_search (no LM, CUDA events over repeated launches), the frames
  kernel's achieved bandwidth against the bytes it must move, and the card's name and power limit read in the same run.

    python profiles/ctc_beam_bench.py [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import MODEL, V, synth_wave  # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still reported, without the power limit
        q = "unavailable (%s)" % e
    return name, q


def _timed(fn, reps):
    """Median milliseconds of fn() over reps calls (CUDA events; fn ends with its own synchronisation where it reads back)."""
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bsz", type=int, default=24)
    ap.add_argument("--seconds", type=float, default=10.0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    dev = torch.device("cuda:0")

    from espresso_b200 import ops
    from espresso_b200.data.asr_dictionary import AsrDictionary
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel
    from espresso_b200.models.lstm_lm import LSTMLanguageModelEspresso, LSTMLanguageModelEspressoConfig
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = AsrDictionary(enable_bos=True)
    for i in range(V - 4):
        d.add_symbol("u%d" % i)
    assert len(d) == V

    class _Task:
        feat_dim, feat_in_channels, target_dictionary = 80, 1, d

    torch.manual_seed(5)
    cfg = SpeechTransformerConfig.from_dict(dict(dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                                                 layernorm_embedding=True, max_source_positions=3600, encoder=MODEL))
    model = SpeechTransformerEncoderModel.build_model(cfg, _Task()).finalize_(dev)
    model.frontend = OnTheFlyFbank(np.full(80, 15.0), np.full(80, 4.0))
    model.eval()
    lm = LSTMLanguageModelEspresso.build_model(LSTMLanguageModelEspressoConfig(
        dropout=0.0, decoder_embed_dim=800, decoder_hidden_size=800, decoder_layers=4, decoder_out_embed_dim=800, share_embed=True),
        _Task()).finalize_(dev)

    B, n = args.bsz, int(args.seconds * 16000)
    rs = np.random.RandomState(3)
    wave = torch.from_numpy(np.stack([synth_wave(rs, n) for _ in range(B)])).to(dev)
    lens = torch.full((B,), n, dtype=torch.int32)
    sample = {"net_input": {"src_tokens": wave, "src_lengths": lens.to(dev), "src_lengths_cpu": lens.long()}}
    audio_s = B * args.seconds
    out = {}
    with torch.no_grad():
        net = model(**sample["net_input"])
        torch.cuda.synchronize()
        enc_ms = _timed(lambda: model(**sample["net_input"]), args.reps)
        logits, T_enc = net["b200_out"], net["src_lengths"][0]
        Tp = logits.shape[1]
        runs = {}
        for beam, with_lm in [(1, False), (10, False), (60, False), (10, True), (60, True)]:
            dec = CTCDecoder(d, beam_size=beam, lm_model=lm if with_lm else None, lm_weight=0.47)
            if dec.greedy:
                fn = lambda: dec._greedy(logits, V, T_enc.tolist())  # noqa: E731
            else:
                fn = lambda: dec.search(logits, V, T_enc)  # noqa: E731
            fn()
            torch.cuda.synchronize()
            ms = _timed(fn, args.reps if not with_lm else max(2, args.reps // 2))
            key = "greedy" if dec.greedy else ("beam%d%s" % (beam, "_lstm_lm" if with_lm else ""))
            runs[key] = {"search_ms": round(ms, 3), "rtf": round((enc_ms + ms) / 1000.0 / audio_s, 6)}
        # per-kernel times of the no-LM path at beam 10 / 60 (K = beam)
        lens_d = T_enc.to(dtype=torch.int32)
        kern = {}
        for beam in (10, 60):
            fr = ops.ctc_beam_frames(logits, V, lens_d, beam, 0, 1, 2, 3)
            ws = ops.ctc_beam_workspace(B, Tp, beam, dev)
            reps = 20
            f_ms = _timed(lambda: [ops.ctc_beam_frames(logits, V, lens_d, beam, 0, 1, 2, 3) for _ in range(reps)], 3) / reps
            s_ms = _timed(lambda: [ops.ctc_beam_search(logits, V, lens_d, fr, beam, float(beam), 0, Tp, ws, eos=2)
                                   for _ in range(reps)], 3) / reps
            rows = int(lens_d.sum())
            nbytes = rows * V * 2 + rows * (4 + 4 + 8 * beam)  # logits read once + lse, lp_blank, top tokens / lp written
            kern["beam%d" % beam] = {"frames_ms": round(f_ms, 4), "search_ms": round(s_ms, 4), "frames_bytes": nbytes,
                                     "frames_GBps": round(nbytes / (f_ms * 1e-3) / 1e9, 1),
                                     "frames_share_of_3.35TBps": round(nbytes / (f_ms * 1e-3) / 3.35e12, 3)}
    name, power = _card()
    out.update(card=name, power_limit_and_max_sm_clock=power, bsz=B, utt_seconds=args.seconds, encoder_frames=Tp, vocab=V,
               encoder_ms=round(enc_ms, 3), decode=runs, kernels=kern)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
