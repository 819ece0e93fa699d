"""CTC decoding with an ARPA n-gram LM on the benchmarked Conformer-CTC (17 x 512, V = 5004, random initialisation), bsz
24 x 10 s utterances as in profiles/ctc_beam_bench.py.  Synthetic LMs are generated from a seed: a word 3-gram and
4-gram over 200 000 words (n-grams taken from a Zipf corpus, so every context is listed; probabilities and backoffs
random) with a lexicon spelling each word in 2-5 pieces (every 7th word with a second spelling, every 11th a homograph
of the word before), and a piece 4-gram for lexicon-free decoding.  Prints one JSON line: ARPA load time and table bytes
per LM, search milliseconds per batch (CUDA events, including the device-to-host copy of the results) at beam 10 and 60
(K = beam), lexicon-free and through the lexicon, next to the LSTM-LM path in the same run, and the card's name and power
limit read in the same run.

    python profiles/ctc_ngram_bench.py [--reps 5] [--words 200000]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from bench import MODEL, V, synth_wave  # noqa: E402
from ctc_beam_bench import _card, _timed  # noqa: E402


def synth_arpa(path, words, order, n_tokens, seed):
    """n-grams of a Zipf corpus over `words` (sentences of 1-30 words between <s> and </s>), random log10 probabilities
    and backoffs, written as ARPA."""
    rs = np.random.RandomState(seed)
    nw = len(words)
    p = 1.0 / np.arange(1, nw + 1) ** 1.1
    p /= p.sum()
    toks = rs.choice(nw, size=n_tokens, p=p).astype(np.int64) + 3  # 0 <s>, 1 </s>, 2 <unk>
    lens = rs.randint(1, 31, size=n_tokens // 15 + 1)
    ends = np.cumsum(lens)
    ends = ends[ends < n_tokens]
    sent = np.split(toks, ends)
    flat = np.concatenate([np.concatenate([[0], s, [1]]) for s in sent])
    sid = np.concatenate([np.full(len(s) + 2, i) for i, s in enumerate(sent)])
    vocab = ["<s>", "</s>", "<unk>"] + list(words)
    sections = []
    for k in range(1, order + 1):
        if k == 1:
            g = np.arange(len(vocab))[:, None]
        else:
            n = len(flat) - k + 1
            ok = sid[:n] == sid[k - 1:]
            win = np.stack([flat[i:i + n] for i in range(k)], 1)[ok]
            g = np.unique(win, axis=0)
        lp = -rs.uniform(0.5, 6.0, size=len(g))
        if k == 1:
            lp[0] = -99.0
        bo = -rs.uniform(0.0, 1.0, size=len(g))
        cols = [" ".join(vocab[i] for i in row) for row in g.tolist()]
        if k < order:
            lines = ["%.6f\t%s\t%.6f" % (a, c, b) for a, c, b in zip(lp, cols, bo)]
        else:
            lines = ["%.6f\t%s" % (a, c) for a, c in zip(lp, cols)]
        sections.append(lines)
    with open(path, "w") as f:
        f.write("\\data\\\n" + "".join("ngram %d=%d\n" % (k + 1, len(s)) for k, s in enumerate(sections)))
        for k, s in enumerate(sections):
            f.write("\n\\%d-grams:\n" % (k + 1))
            f.write("\n".join(s))
            f.write("\n")
        f.write("\n\\end\\\n")
    return sum(len(s) for s in sections)


def synth_lexicon(path, words, pieces, seed):
    rs = np.random.RandomState(seed)
    out, prev = [], None
    for i, w in enumerate(words):
        sp = " ".join(rs.choice(pieces, size=rs.randint(2, 6)))
        if i % 11 == 10 and prev is not None:
            sp = prev
        out.append("%s\t%s\n" % (w, sp))
        if i % 7 == 6:
            out.append("%s\t%s\n" % (w, " ".join(rs.choice(pieces, size=rs.randint(2, 6)))))
        prev = sp
    with open(path, "w") as f:
        f.writelines(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--bsz", type=int, default=24)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--words", type=int, default=200000)
    ap.add_argument("--tokens", type=int, default=3000000)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    dev = torch.device("cuda:0")

    from espresso_b200.data.asr_dictionary import AsrDictionary
    from espresso_b200.data.frontend import OnTheFlyFbank
    from espresso_b200.models import NgramLanguageModel, SpeechTransformerConfig, SpeechTransformerEncoderModel
    from espresso_b200.models.lstm_lm import LSTMLanguageModelEspresso, LSTMLanguageModelEspressoConfig
    from espresso_b200.tools.ctc_decoder import CTCDecoder

    d = AsrDictionary(enable_bos=True)
    for i in range(V - 4):
        d.add_symbol("u%d" % i)
    pieces = ["u%d" % i for i in range(V - 4)]

    class _Task:
        feat_dim, feat_in_channels, target_dictionary = 80, 1, d

    torch.manual_seed(5)
    cfg = SpeechTransformerConfig.from_dict(dict(dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                                                 layernorm_embedding=True, max_source_positions=3600, encoder=MODEL))
    model = SpeechTransformerEncoderModel.build_model(cfg, _Task()).finalize_(dev)
    model.frontend = OnTheFlyFbank(np.full(80, 15.0), np.full(80, 4.0))
    model.eval()
    lstm = LSTMLanguageModelEspresso.build_model(LSTMLanguageModelEspressoConfig(
        dropout=0.0, decoder_embed_dim=800, decoder_hidden_size=800, decoder_layers=4, decoder_out_embed_dim=800, share_embed=True),
        _Task()).finalize_(dev)

    B, n = args.bsz, int(args.seconds * 16000)
    rs = np.random.RandomState(3)
    wave = torch.from_numpy(np.stack([synth_wave(rs, n) for _ in range(B)])).to(dev)
    lens = torch.full((B,), n, dtype=torch.int32)
    words = ["w%d" % i for i in range(args.words)]
    out, lms = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        lex = os.path.join(tmp, "lexicon.txt")
        synth_lexicon(lex, words, pieces, seed=1)
        for name, vocab, order, seed in (("word3", words, 3, 1), ("word4", words, 4, 2), ("piece4", pieces, 4, 3)):
            path = os.path.join(tmp, name + ".arpa")
            n_gram = synth_arpa(path, vocab, order, args.tokens, seed)
            t0 = time.perf_counter()
            lm = NgramLanguageModel.from_arpa(path)
            load_s = time.perf_counter() - t0
            lm.to(dev)
            torch.cuda.synchronize()
            lms[name] = lm
            out[name] = {"ngrams": n_gram, "arpa_mb": round(os.path.getsize(path) / 1e6, 1), "load_s": round(load_s, 3),
                         "table_bytes": lm.table_bytes}
        with torch.no_grad():
            net = model(src_tokens=wave, src_lengths=lens.to(dev), src_lengths_cpu=lens.long())
            logits, T_enc = net["b200_out"], net["src_lengths"][0]
            runs = {}
            for beam in (10, 60):
                cases = [("lstm_lm", dict(lm_model=lstm, lm_weight=0.47)),
                         ("piece4_lexicon_free", dict(lm_model=lms["piece4"], lm_weight=0.47)),
                         ("word3_lexicon", dict(lm_model=lms["word3"], lm_weight=2.0, word_score=-1.0, lexicon=lex)),
                         ("word4_lexicon", dict(lm_model=lms["word4"], lm_weight=2.0, word_score=-1.0, lexicon=lex))]
                for key, kw in cases:
                    dec = CTCDecoder(d, beam_size=beam, **kw)
                    fn = lambda: dec.search(logits, V, T_enc)  # noqa: E731
                    fn()
                    torch.cuda.synchronize()
                    runs["beam%d_%s" % (beam, key)] = round(_timed(fn, args.reps if key != "lstm_lm" else max(2, args.reps // 2)), 3)
    name, power = _card()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=power, bsz=B, utt_seconds=args.seconds,
                          encoder_frames=int(logits.shape[1]), vocab=V, lms=out, search_ms=runs)))


if __name__ == "__main__":
    main()
