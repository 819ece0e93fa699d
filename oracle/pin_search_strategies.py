"""Pin oracle/search_strategies.generate against the REAL reference and write tests/golden/search_strategies.npz.

Runs only where the reference tree is present (imported through oracle/refshim):
    python -m oracle.pin_search_strategies
The reference's SequenceGenerator (Espresso's fairseq, with lm_model / lm_weight / eos_factor) runs with
search.DiverseBeamSearch, search.DiverseSiblingsSearch, search.Sampling (deterministic cases: top-p below the top-1
probability, top-k = 1), no_repeat_ngram_size and prefix_tokens on the prefix-dependent table
models of oracle/pin_against_reference.py::pin_beam; the oracle must give the same hypotheses (tokens exact, scores 1e-5).

N-gram blocking: the reference blocks through its CUDA extension (fairseq/clib/cuda/ngram_repeat_block_cuda_kernel.cu),
which compares the window ending at the current step.  Its CPU fallback, NGramRepeatBlock._no_repeat_ngram, states the
same rule for a token history of step + 1 columns (the reference's TestRepeatNgramBlocking checks the two against each
other that way), but the generator hands it the whole max_len + 2 buffer, whose trailing columns are pad, so on the CPU
it would block nothing.  The pin therefore hands the fallback tokens[:, :step + 1], i.e. runs the extension's rule.
"""
import os
import sys

import numpy as np
import torch

from oracle import refshim
from oracle.pin_against_reference import _table_lprobs

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
PAD, EOS, UNK = 1, 2, 3

# name -> options; every case: max_len_b 12, min_len 2, unk penalty 0.3, src_len 7, model max positions 40
CASES = [
    dict(seed=31, beam=4, bsz=3, V=11, groups=2, strength=0.5),
    dict(seed=32, beam=6, bsz=2, V=13, groups=3, strength=1.3, lm=0.4, eos_factor=1.5),
    dict(seed=33, beam=4, bsz=3, V=9, groups=2, strength=0.0),
    dict(seed=34, beam=3, bsz=3, V=10, rate=0.5),
    dict(seed=35, beam=4, bsz=2, V=12, rate=1.1, lm=0.3, lenpen=0.6),
    dict(seed=60, beam=3, bsz=2, V=6, ngram=2),
    dict(seed=67, beam=4, bsz=2, V=7, ngram=3, lm=0.5, eos_factor=1.5),
    dict(seed=38, beam=5, bsz=3, V=9, ngram=2, lm=0.47),
    dict(seed=60, beam=3, bsz=2, V=6, ngram=3, eos_factor=2.0),
    dict(seed=40, beam=3, bsz=4, V=10, prefix=[[4, 5, 6], [7, PAD, 4], [5, EOS, PAD], [PAD, PAD, PAD]]),
    dict(seed=41, beam=4, bsz=3, V=9, prefix=[[4, EOS], [4, PAD], [PAD, PAD]], lm=0.3),
    dict(seed=42, beam=4, bsz=3, V=11, prefix=[[6, 6], [4, EOS], [PAD, 5]], ngram=2, groups=2, strength=0.7),
    dict(seed=43, beam=3, bsz=2, V=10, prefix=[[5, 7, 6, 4], [8, 8, PAD, PAD]], ngram=2, rate=0.4, eos_factor=1.5),
    # sampling, deterministic: top-p below every row's top-1 probability (>= 1 / V), and top-k = 1
    dict(seed=44, beam=3, bsz=3, V=9, topp=0.05),
    dict(seed=45, beam=4, bsz=2, V=12, topk=1, lm=0.3, ngram=2),
    dict(seed=46, beam=2, bsz=3, V=10, topp=0.02, prefix=[[6, PAD], [7, EOS], [PAD, PAD]]),
]


def case_kwargs(c):
    """The generator keywords of case c (oracle/search_strategies.generate and espresso_b200's SequenceGenerator)."""
    kw = dict(beam_size=c["beam"], max_len_a=0.0, max_len_b=12, min_len=2, len_penalty=c.get("lenpen", 1.0), unk_penalty=0.3,
              eos_factor=c.get("eos_factor"), no_repeat_ngram_size=c.get("ngram", 0))
    if "groups" in c:
        kw.update(diverse_beam_groups=c["groups"], diverse_beam_strength=c["strength"])
    if "rate" in c:
        kw.update(diversity_rate=c["rate"])
    if "topp" in c or "topk" in c:
        kw.update(sampling=True, sampling_topk=c.get("topk", -1), sampling_topp=c.get("topp", -1.0))
    return kw


def lprobs_fn(c):
    def fn(step, tokens, ro):
        lp = _table_lprobs(c["seed"], c["V"], step, tokens)
        if c.get("lm") is not None:
            lp = lp + c["lm"] * _table_lprobs(c["seed"] + 1000, c["V"], step, tokens)
        return lp
    return fn


def pin():
    import argparse

    from fairseq import search
    from fairseq.ngram_repeat_block import NGramRepeatBlock
    from fairseq.sequence_generator import SequenceGenerator
    from tests import utils as ref_test_utils

    from oracle import search_strategies as OS

    fallback = NGramRepeatBlock._no_repeat_ngram
    NGramRepeatBlock._no_repeat_ngram = lambda self, tokens, lprobs, bsz, beam, step: fallback(
        self, tokens[:, : step + 1], lprobs, bsz, beam, step)
    out = {"n_cases": np.int64(len(CASES))}
    n_h = 0
    for ci, c in enumerate(CASES):
        V, seed = c["V"], c["seed"]
        d = ref_test_utils.dummy_dictionary(vocab_size=V - 4)
        assert len(d) == V and d.pad() == PAD and d.eos() == EOS and d.unk() == UNK

        class Dec(ref_test_utils.TestIncrementalDecoder):
            def forward(self, prev_output_tokens, encoder_out=None, incremental_state=None):
                return _table_lprobs(seed, V, prev_output_tokens.size(1) - 1, prev_output_tokens)[:, None, :], {"attn": [None]}

            def get_normalized_probs(self, net_output, log_probs, _):
                return net_output[0]

        class LM:
            def __init__(self):
                self.decoder = self

            def eval(self):
                return self

            def reorder_incremental_state_scripting(self, state, order):
                pass

            def __call__(self, tokens, incremental_state=None):
                return (_table_lprobs(seed + 1000, V, tokens.size(1) - 1, tokens)[:, None, :], None)

            def get_normalized_probs(self, net_output, log_probs, sample=None):
                return net_output[0]

        if "groups" in c:
            strategy = search.DiverseBeamSearch(d, c["groups"], c["strength"])
        elif "rate" in c:
            strategy = search.DiverseSiblingsSearch(d, c["rate"])
        elif "topp" in c or "topk" in c:
            strategy = search.Sampling(d, sampling_topk=c.get("topk", -1), sampling_topp=c.get("topp", -1.0))
        else:
            strategy = None
        kw = case_kwargs(c)
        args = argparse.Namespace(beam_probs=[], max_decoder_positions=40)
        model = ref_test_utils.TestModel(ref_test_utils.TestEncoder(args, d), Dec(args, d))
        gen = SequenceGenerator([model], d, beam_size=kw["beam_size"], max_len_a=0.0, max_len_b=12, min_len=2,
                                len_penalty=kw["len_penalty"], unk_penalty=0.3, lm_model=LM() if c.get("lm") is not None else None,
                                lm_weight=c.get("lm") or 1.0, eos_factor=kw["eos_factor"], no_repeat_ngram_size=kw["no_repeat_ngram_size"],
                                search_strategy=strategy)
        src = torch.full((c["bsz"], 7), 5, dtype=torch.long)
        src[:, -1] = EOS
        sample = {"net_input": {"src_tokens": src, "src_lengths": torch.full((c["bsz"],), 7)}}
        prefix = torch.tensor(c["prefix"], dtype=torch.long) if "prefix" in c else None
        ref = gen.generate([model], sample, prefix_tokens=prefix)
        ours = OS.generate(lprobs_fn(c), c["bsz"], 7, V, PAD, UNK, EOS, model_max_len=40, prefix_tokens=prefix, **kw)
        for b, (rh, oh) in enumerate(zip(ref, ours)):
            assert len(rh) == len(oh), (ci, b, len(rh), len(oh))
            for k, (r_, o_) in enumerate(zip(rh, oh)):
                assert r_["tokens"].tolist() == o_["tokens"].tolist(), (ci, b, k, r_["tokens"].tolist(), o_["tokens"].tolist())
                assert abs(float(r_["score"]) - float(o_["score"])) < 1e-5, (ci, b, k)
                assert (r_["positional_scores"] - o_["positional_scores"]).abs().max() < 1e-5, (ci, b, k)
                out["c%d_b%d_k%d_tokens" % (ci, b, k)] = r_["tokens"].numpy()
                out["c%d_b%d_k%d_score" % (ci, b, k)] = np.float32(float(r_["score"]))
                n_h += 1
            out["c%d_b%d_n" % (ci, b)] = np.int64(len(rh))
        print("case %d %s: %d hypotheses agree" % (ci, {k: v for k, v in c.items() if k != "prefix"}, sum(len(h) for h in ref)))
    NGramRepeatBlock._no_repeat_ngram = fallback
    np.savez_compressed(os.path.join(GOLDEN, "search_strategies.npz"), **out)
    print("search strategies: %d hypotheses pinned" % n_h)


if __name__ == "__main__":
    refshim.activate()
    torch.manual_seed(0)
    pin()
    sys.exit(0)
