"""CTC prefix beam search fused with the Transformer LM of bench.py's decode (6 x 512, 8 heads, FFN 2048, V = 5004,
random initialisation) on the logits of the benchmarked Conformer-CTC: bsz 24 x 10 s utterances (250 encoder frames),
the batch of the LSTM-LM rows in DESIGN.md §7, at beam 10 and 60.  Prints one JSON line: per beam the search
milliseconds per batch (median of --reps, CUDA events; the search includes the final device-to-host copy), native
launches per frame (esp_launch_count over one search, minus frames / finalize, over T'), the frame-slot KV cache's bytes
(T' + 1 slots x N rows x 2d x 2 B x layers, allocated as such), and the card's name and power limit read in the same run.

    python profiles/ctc_transformer_lm_bench.py [--reps 5]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench import MODEL, V, synth_wave  # noqa: E402
from ctc_beam_bench import _card, _timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bsz", type=int, default=24)
    ap.add_argument("--seconds", type=float, default=10.0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    dev = torch.device("cuda:0")

    from espresso_b200 import lib
    from espresso_b200.data.asr_dictionary import AsrDictionary
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import SpeechTransformerConfig, SpeechTransformerEncoderModel
    from espresso_b200.models.transformer_lm import TransformerLanguageModel
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = AsrDictionary(enable_bos=True)
    for i in range(V - 4):
        d.add_symbol("u%d" % i)

    class _Task:
        feat_dim, feat_in_channels, target_dictionary = 80, 1, d

    torch.manual_seed(5)
    cfg = SpeechTransformerConfig.from_dict(dict(dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                                                 layernorm_embedding=True, max_source_positions=3600, encoder=MODEL))
    model = SpeechTransformerEncoderModel.build_model(cfg, _Task()).finalize_(dev)
    model.frontend = OnTheFlyFbank(np.full(80, 15.0), np.full(80, 4.0))
    model.eval()
    lm = TransformerLanguageModel(d, embed_dim=512, ffn_embed_dim=2048, layers=6, attention_heads=8,
                                  max_target_positions=1024).finalize_(dev)

    B, n = args.bsz, int(args.seconds * 16000)
    rs = np.random.RandomState(3)
    wave = torch.from_numpy(np.stack([synth_wave(rs, n) for _ in range(B)])).to(dev)
    lens = torch.full((B,), n, dtype=torch.int32)
    sample = {"net_input": {"src_tokens": wave, "src_lengths": lens.to(dev), "src_lengths_cpu": lens.long()}}
    runs = {}
    with torch.no_grad():
        net = model(**sample["net_input"])
        logits, T_enc = net["b200_out"], net["src_lengths"][0]
        Tp = logits.shape[1]
        for beam in (10, 60):
            dec = CTCDecoder(d, beam_size=beam, lm_model=lm, lm_weight=0.47)
            dec.search(logits, V, T_enc)
            torch.cuda.synchronize()
            c0 = lib.launch_count()
            dec.search(logits, V, T_enc)
            launches = lib.launch_count() - c0
            ms = _timed(lambda: dec.search(logits, V, T_enc), args.reps)
            N = B * beam
            runs["beam%d_transformer_lm" % beam] = {
                "search_ms": round(ms, 3), "search_ms_per_frame": round(ms / Tp, 4),
                "launches_per_frame": round((launches - 2) / Tp, 2),  # minus frames and finalize
                "kv_cache_bytes": (Tp + 1) * N * 2 * lm.cfg["embed_dim"] * 2 * lm.cfg["layers"]}
    name, power = _card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=power, bsz=B, utt_seconds=args.seconds, encoder_frames=Tp,
                          vocab=V, lm="transformer_lm 6 x 512, 8 heads, FFN 2048", reps=args.reps, decode=runs)))


if __name__ == "__main__":
    main()
