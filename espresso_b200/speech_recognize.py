"""The decode-and-score loop of the reference's `speech_recognize.py` as a library call (espresso/speech_recognize.py:60-400;
host logic around the search kernels -- no command line, no config system):

    out = recognize(task, models, subset="test", gen_args=Namespace(beam=5, lm_weight=0.47, eos_factor=1.5, ...),
                    lms=[subword_lm] | [word_lm] | [subword_lm, word_lm], max_tokens=12000, device="cuda:0")
    out["scorer"].wer()      # (WER %, sub %, ins %, del %)

It wraps word-level LMs the way the reference does (:134-160: a word LM alone -> TensorizedLookaheadLanguageModel, a word LM
behind a subword LM -> MultiLevelLanguageModel), builds the decoder the task picks for the criterion (beam search with LM
fusion, CTC greedy, transducer greedy / beam search), walks the subset in its stored order through the task's batch iterator,
prints `T-<utt>` / `H-<utt>\\t<hyp>\\t<score in base 2>` lines like the reference (:262-290) and feeds the best hypothesis of
every utterance to a `Scorer` (sub-word and word error counts, aligned output).  With print_alignment on an attention model
(criterion neither ctc_loss nor transducer_loss) it also plots the best hypothesis's encoder attention over the utterance's
non-padded frames to <results_path>/attn_plots/<utt_id>.pdf (:212-221,270,302-314)."""
import math
import os
import time
from argparse import Namespace

import torch

from . import ops as _ops
from .data import flac as _flac
from .tools.utils import plot_attention
from .tools.wer import Scorer


def wrap_language_models(lms, dictionary, gen_args):
    """-> the single LM object the generator fuses (or None)."""
    from .models import MultiLevelLanguageModel, TensorizedLookaheadLanguageModel

    lms = [m for m in (lms or []) if m is not None]
    if not lms:
        return None
    assert len(lms) in (1, 2), "one LM, or a subword LM followed by a word LM"
    g = lambda k, d: getattr(gen_args, k, d)  # noqa: E731
    last = lms[-1]
    if getattr(last, "is_wordlm", False):
        if len(lms) == 2:  # the subword LM comes first
            return MultiLevelLanguageModel(last, lms[0], subwordlm_weight=g("subwordlm_weight", 0.8),
                                           oov_penalty=g("oov_penalty", 1e-4), open_vocab=not g("disable_open_vocab", False))
        return TensorizedLookaheadLanguageModel(last, dictionary, oov_penalty=g("oov_penalty", 1e-4),
                                                open_vocab=not g("disable_open_vocab", False))
    assert len(lms) == 1, "two LMs are only combined when the second one is a word LM"
    return last


def _to_device(x, device):
    if isinstance(x, _flac.PackedFlac):  # FLAC batch: uploaded compressed, decoded on the device
        return _flac.to_device(x, device)[0]
    if torch.is_tensor(x):
        return x.to(device, non_blocking=True)
    if isinstance(x, dict):
        return {k: _to_device(v, device) for k, v in x.items()}
    return x


def recognize(task, models, subset=None, gen_args=None, lms=None, max_tokens=12000, max_sentences=None, device=None, nbest=1,
              wer_output_filter=None, quiet=True, out=None, num_shards=1, shard_id=0, print_alignment=False, results_path=None):
    """Decode `subset` with `models` (an ensemble list) and score it.  Returns {"scorer", "num_sentences", "num_tokens",
    "seconds", "lines"}; `lines` are the reference's T- / H- output lines (also written to `out` when given).
    print_alignment: attention plots of the best hypotheses under results_path (attention models only; the CTC and
    transducer decoders keep their own meaning of gen_args.print_alignment)."""
    gen_args = gen_args if gen_args is not None else Namespace()
    # espresso/speech_recognize.py:43-44
    assert not getattr(gen_args, "sampling", False) or nbest == getattr(gen_args, "beam", 5), \
        "--sampling requires --nbest to be equal to --beam"
    prefix_size = getattr(gen_args, "prefix_size", 0) or 0
    subset = subset or task.cfg.gen_subset
    dictionary = task.target_dictionary
    dev = torch.device(device) if device is not None else next(models[0].parameters()).device
    lm = wrap_language_models(lms, dictionary, gen_args)
    extra = {"lm_model": lm, "lm_weight": getattr(gen_args, "lm_weight", 0.0), "eos_factor": getattr(gen_args, "eos_factor", None)}
    save_attention_plot = bool(print_alignment) and task.cfg.criterion_name not in ("transducer_loss", "ctc_loss")
    if save_attention_plot:
        if results_path is None:
            raise ValueError("print_alignment saves attention plots under results_path; pass results_path")
        extra["print_alignment"] = True
    generator = task.build_generator(models, gen_args, extra_gen_cls_kwargs=extra)
    if subset not in task.datasets:
        task.load_dataset(subset)
    itr = task.get_batch_iterator(task.dataset(subset), max_tokens=max_tokens, max_sentences=max_sentences, num_shards=num_shards,
                                  shard_id=shard_id).next_epoch_itr(shuffle=False)
    scorer = Scorer(dictionary, wer_output_filter=wer_output_filter)
    strip = {dictionary.eos(), dictionary.pad()}
    if getattr(dictionary, "bos_index", None) is not None and getattr(dictionary, "enable_bos", True):
        strip.add(dictionary.bos())
    lines, n_sent, n_tok, t0 = [], 0, 0, time.perf_counter()

    def emit(s):
        lines.append(s)
        if out is not None and not quiet:
            print(s, file=out)

    for m in models:
        m.eval()
    for sample in itr:
        if not sample or "net_input" not in sample:
            continue  # a padding batch of the sharded iterator
        s_dev = _to_device(sample, dev)
        with torch.no_grad():
            # the first prefix_size target tokens are forced (espresso/speech_recognize.py:246-248)
            kw = {"prefix_tokens": s_dev["target"][:, :prefix_size]} if prefix_size > 0 else {}
            hypos = generator.generate(models, s_dev, **kw)
        n_tok += sum(len(h[0]["tokens"]) for h in hypos)
        if save_attention_plot:  # non-padded encoder frames of every utterance
            src, lens = s_dev["net_input"]["src_tokens"], s_dev["net_input"]["src_lengths"]
            if src.dim() == 2 and src.is_floating_point():  # raw waveforms: sample counts -> fbank frames
                lens = _ops.num_frames(lens)
            out_lens = models[0].encoder.output_lengths(lens).tolist()
        for i in range(len(sample["id"])):
            utt_id = sample["utt_id"][i]
            has_target = sample.get("text") is not None
            if has_target:
                target_str = dictionary.wordpiece_encode(sample["text"][i])
                emit("T-%s\t%s" % (utt_id, sample["text"][i]))
            for j, hypo in enumerate(hypos[i][:nbest]):
                hypo_str = dictionary.string(hypo["tokens"].int().cpu(), bpe_symbol=None, extra_symbols_to_ignore=strip)
                emit("H-%s\t%s\t%s" % (utt_id, dictionary.wordpiece_decode(hypo_str), float(hypo["score"]) / math.log(2)))
                if j == 0:
                    if save_attention_plot and hypo["attention"] is not None:  # src_len x tgt_len
                        save_dir = os.path.join(results_path, "attn_plots")
                        os.makedirs(save_dir, exist_ok=True)
                        plot_attention(hypo["attention"][: int(out_lens[i])].float().cpu(), dictionary.wordpiece_decode(hypo_str),
                                       utt_id, save_dir)
                    scorer.add_prediction(utt_id, hypo_str)
                    if has_target:
                        scorer.add_evaluation(utt_id, target_str, hypo_str)
        n_sent += int(sample.get("nsentences", len(sample["id"])))
    return {"scorer": scorer, "num_sentences": n_sent, "num_tokens": n_tok, "seconds": time.perf_counter() - t0, "lines": lines}
