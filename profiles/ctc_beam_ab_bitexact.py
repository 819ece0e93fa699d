"""Do two builds of the library decode the same?  Replays the no-LM and LSTM-LM CTC prefix beam search cases of
tests/test_gpu_ctc_beam.py and the lexicon-free and lexicon n-gram cases of tests/test_gpu_ngram.py (same shapes, seeds
and decoder options) through the in-tree library and through --other-lib on the same inputs and compares tokens,
lengths, scores and frames bit for bit.

    python profiles/ctc_beam_ab_bitexact.py --other-lib PATH

PATH is another build of libespresso_b200.so, e.g. the parent commit's: `git worktree add /tmp/parent HEAD~1 &&
make -C /tmp/parent/espresso_b200/csrc`.  Exits non-zero on any difference."""
import argparse
import ctypes
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from espresso_b200 import lib  # noqa: E402
from test_ctc_beam_search import _dict, _lstm_lm  # noqa: E402
from test_gpu_ctc_beam import _decoder, _repeat_heavy, _x  # noqa: E402
from test_gpu_ngram import _lex_decoder, _lexicon, _sym_lm  # noqa: E402

DEV = torch.device("cuda:0")


def cases():
    """(name, decoder factory, logits, lens, V) as the GPU tests build them."""
    for beam in (1, 4, 16, 60):
        yield ("no_lm_ragged_beam%d" % beam, lambda beam=beam: _decoder(40, beam, nbest=min(beam, 3), print_alignment=True,
                                                                        word_score=0.25),
               _x(4, 50, 40, seed=beam, scale=2.0), torch.tensor([50, 33, 1, 0]), 40)
    for beam, K, thr, blank in [(16, 5, None, 0), (16, 16, 2.0, 0), (8, 8, None, 7), (60, 12, 4.0, 5)]:
        yield ("no_lm_options_%d_%d_%s_%d" % (beam, K, thr, blank),
               lambda beam=beam, K=K, thr=thr, blank=blank: _decoder(48, beam, blank=blank, beam_size_token=K, beam_threshold=thr,
                                                                     nbest=3),
               _x(3, 40, 48, seed=beam + K + blank, scale=2.5), torch.tensor([40, 17, 29]), 48)
    for beam in (4, 16):
        yield ("repeat_heavy_beam%d" % beam, lambda beam=beam: _decoder(24, beam, nbest=2, print_alignment=True),
               _repeat_heavy(4, 60, 24, seed=beam), torch.tensor([60, 59, 31, 2]), 24)
    yield ("recipe_shape", lambda: _decoder(5004, 10, nbest=2), _repeat_heavy(24, 875, 5004, seed=11, peak=6.0),
           torch.tensor([875 - 13 * b for b in range(24)]), 5004)
    for beam, lm_blank in [(4, False), (16, True), (60, False)]:
        def make(beam=beam, lm_blank=lm_blank):
            lm = _lstm_lm(_dict(n_sym=32, bos=not lm_blank), seed=beam, hidden=32).finalize_(DEV, dtype=torch.float32)
            return _decoder(36, beam, lm=lm, lm_weight=0.47, word_score=0.6, nbest=3, print_alignment=True)
        yield ("lstm_lm_beam%d_blank%s" % (beam, lm_blank), make, _x(3, 30, 36, seed=100 + beam, scale=2.0),
               torch.tensor([30, 21, 0]), 36)
    tmp = tempfile.mkdtemp()
    for beam, order, case in [(4, 2, "random"), (16, 3, "repeat"), (60, 4, "random")]:
        def make(beam=beam, order=order):
            from pathlib import Path

            from espresso_b200.tools.ctc_decoder import CTCDecoder

            d = _dict(n_sym=24)
            _, lm = _sym_lm(Path(tmp), d, order, seed=beam)
            return CTCDecoder(d, blank_idx=0, beam_size=beam, lm_model=lm, lm_weight=0.9, word_score=0.4, nbest=3,
                              print_alignment=True)
        yield ("ngram_free_beam%d_order%d" % (beam, order), make,
               _x(4, 40, 28, seed=beam, scale=2.0) if case == "random" else _repeat_heavy(4, 40, 28, seed=beam),
               torch.tensor([40, 23, 1, 0]), 28)
    for beam, order, case in [(4, 2, "random"), (16, 3, "repeat"), (40, 3, "random")]:
        def make(beam=beam, order=order):
            from pathlib import Path

            d = _dict(n_sym=16)
            return _lex_decoder(Path(tmp), d, _lexicon(d, 40, seed=beam), order, beam, beam, lm_weight=0.8, word_score=-0.3,
                                nbest=3, print_alignment=True)[1]
        yield ("ngram_lexicon_beam%d_order%d" % (beam, order), make,
               _x(4, 36, 20, seed=beam, scale=2.0) if case == "random" else _repeat_heavy(4, 36, 20, seed=beam),
               torch.tensor([36, 20, 1, 0]), 20)


def run(handle, make, x, lens, V):
    saved = lib._lib
    lib._lib = handle
    try:
        out = make().search(x.to(DEV), V, lens.to(DEV))
    finally:
        lib._lib = saved
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other-lib", required=True)
    args = ap.parse_args()
    mine = lib.load()
    other = ctypes.CDLL(os.path.abspath(args.other_lib))
    for name, (res, argtypes) in lib.SIGNATURES.items():  # an older build lacks the newer entry points
        if hasattr(other, name):
            fn = getattr(other, name)
            fn.restype, fn.argtypes = res, argtypes
    bad, n = [], 0
    for name, make, x, lens, V in cases():
        a, b = run(mine, make, x, lens, V), run(other, make, x, lens, V)
        for i, (p, q) in enumerate(zip(a, b)):
            if (p is None) != (q is None) or (p is not None and not torch.equal(p.view(torch.int32) if p.dtype == torch.float32 else p,
                                                                                 q.view(torch.int32) if q.dtype == torch.float32 else q)):
                bad.append("%s output %d" % (name, i))
        n += 1
    print(json.dumps({"cases": n, "bit_identical": n - len({b.split(" output")[0] for b in bad}), "differences": bad}))
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
