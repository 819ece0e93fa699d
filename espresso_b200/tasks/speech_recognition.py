"""`speech_recognition_espresso` task: the object the reference hands to models, criterions and generators
(espresso/tasks/speech_recognition.py:272-687).  Host logic only: dictionary set-up (the optional <s> symbol doubles as
the CTC / transducer blank, :324-357), `feat_dim` / `feat_in_channels`, model / criterion construction through the
registries, the generator choice per criterion (:526-596) and validation with word / character error counts
(:598-607, 662-687; error counting restates espresso/tools/wer.py + espresso/tools/utils.py:265-330 as a plain
Levenshtein distance).  Data loading from Kaldi/JSON manifests is out of scope (SURVEY.md §2): the task is built from a
dictionary and a feature dimension, batches come from espresso_b200.data.collate."""
import os
from dataclasses import dataclass
from typing import Optional

from ..data.asr_dictionary import AsrDictionary
from ..registry import CRITERION_REGISTRY, MODEL_REGISTRY, register_task


@dataclass
class SpeechRecognitionEspressoConfig:
    criterion_name: str = "label_smoothed_cross_entropy_v2"  # | "ctc_loss" | "transducer_loss"
    dict: Optional[str] = None
    non_lang_syms: Optional[str] = None
    feat_in_channels: int = 1
    max_source_positions: int = 3600
    max_target_positions: int = 1024
    include_eos_in_transducer_loss: bool = False
    max_num_expansions_per_step: int = 2
    bpe: Optional[str] = None  # how token sequences become words for WER: None (tokens are words) | "sentencepiece" | ...
    seed: int = 1
    # ---- data (espresso/tasks/speech_recognition.py:31-118) ----
    data: Optional[str] = None  # directory (or ":"-separated shards) with {split}.json manifests
    upsample_primary: int = 1
    autoregressive: bool = False
    specaugment_config: Optional[str] = None
    global_cmvn_stats_path: Optional[str] = None
    required_seq_len_multiple: int = 1
    train_subset: str = "train"
    valid_subset: str = "valid"
    gen_subset: str = "test"


def edit_counts(ref, hyp):
    """(errors, len(ref)) with errors = substitutions + insertions + deletions of the best alignment."""
    prev = list(range(len(hyp) + 1))
    for i in range(1, len(ref) + 1):
        cur = [i] + [0] * len(hyp)
        for j in range(1, len(hyp) + 1):
            cur[j] = prev[j - 1] if ref[i - 1] == hyp[j - 1] else 1 + min(prev[j - 1], cur[j - 1], prev[j])
        prev = cur
    return prev[len(hyp)], len(ref)


@register_task("speech_recognition_espresso", dataclass=SpeechRecognitionEspressoConfig)
class SpeechRecognitionEspressoTask:
    def __init__(self, cfg, tgt_dict, feat_dim, word_dict=None):
        self.cfg = cfg
        self.tgt_dict, self.word_dict = tgt_dict, word_dict
        self.feat_dim = feat_dim
        self.feat_in_channels = cfg.feat_in_channels
        self.extra_symbols_to_ignore = {tgt_dict.pad()}  # for validation with WER
        self.blank_symbol = None
        if cfg.criterion_name in ("transducer_loss", "ctc_loss"):
            self.blank_symbol = tgt_dict[tgt_dict.bos()]  # the bos symbol is reserved for blank
            self.extra_symbols_to_ignore.add(tgt_dict.bos())
        self.decoder_for_validation = None
        self.datasets = {}

    @classmethod
    def load_dictionary(cls, filename, enable_bos=False, non_lang_syms=None):
        return AsrDictionary.load(filename, enable_bos=enable_bos, f_non_lang_syms=non_lang_syms)

    @classmethod
    def setup_task(cls, cfg, feat_dim=80, **unused):
        enable_blank = cfg.criterion_name in ("transducer_loss", "ctc_loss")
        tgt_dict = cls.load_dictionary(cfg.dict, enable_bos=enable_blank, non_lang_syms=cfg.non_lang_syms)
        return cls(cfg, tgt_dict, feat_dim)

    @property
    def target_dictionary(self):
        return self.tgt_dict

    @property
    def word_dictionary(self):
        return self.word_dict

    def max_positions(self):
        return (self.cfg.max_source_positions, self.cfg.max_target_positions)

    # ---- data ------------------------------------------------------------------------------------------------
    def load_dataset(self, split, epoch=1, combine=False, **unused):
        """JSON manifest -> AsrDataset (speech_recognition.py:415-468).  Waveform entries stay raw: fbank, global CMVN
        (`global_cmvn_stats_path`, applied by the model's OnTheFlyFbank) and SpecAugment masking run on the device."""
        from ..data.asr_dataset import get_asr_dataset_from_json

        paths = [p for p in (self.cfg.data or "").split(os.pathsep) if p]
        if not paths:
            raise ValueError("task.data is not set")
        if split != self.cfg.train_subset:
            paths = paths[:1]   # validation / test always come from the first shard
        transducer = self.cfg.criterion_name == "transducer_loss"
        self.datasets[split] = ds = get_asr_dataset_from_json(
            paths[(epoch - 1) % len(paths)], split, self.tgt_dict, combine=combine, upsample_primary=self.cfg.upsample_primary,
            shuffle=(split != self.cfg.gen_subset), pad_to_multiple=self.cfg.required_seq_len_multiple,
            autoregressive=self.cfg.autoregressive,
            prepend_bos_as_input_feeding=(transducer and self.cfg.include_eos_in_transducer_loss),
            is_training_set=(split == self.cfg.train_subset), batch_based_on_both_src_tgt=transducer, seed=self.cfg.seed,
            specaugment_config=self.cfg.specaugment_config)
        if split == self.cfg.train_subset and ds.tgt is not None:  # eos / unk counts from the training text (:460-468)
            self.tgt_dict.count[self.tgt_dict.eos()] = len(ds.tgt)
            unk = self.tgt_dict.unk()
            self.tgt_dict.count[unk] = int(sum(int((ds.tgt[i][0] == unk).sum()) for i in range(len(ds.tgt))))
        return ds

    def dataset(self, split):
        if split not in self.datasets:
            raise KeyError("Dataset not loaded: " + split)
        return self.datasets[split]

    def get_batch_iterator(self, dataset, max_tokens=None, max_sentences=None, required_batch_size_multiple=1, seed=1, num_shards=1,
                           shard_id=0, num_workers=2, epoch=1, data_buffer_size=4):
        """fairseq/tasks/fairseq_task.py:231-348: batches are formed once (ordered_indices -> batch_by_size) and frozen;
        the iterator shuffles them per epoch, shards them over ranks and assembles them in background threads."""
        from ..data.iterators import EpochBatchIterator

        dataset.set_epoch(epoch)
        batches = dataset.batch_by_size(dataset.ordered_indices(), max_tokens, max_sentences, required_batch_size_multiple)
        return EpochBatchIterator(dataset, batches, seed=seed, num_shards=num_shards, shard_id=shard_id, num_workers=num_workers,
                                  buffer_size=data_buffer_size, epoch=epoch)

    # ---- construction through the registries ----------------------------------------------------------------
    def build_model(self, model_cfg, arch="speech_transformer_encoder_model", **kw):
        from .. import models  # noqa: F401  (importing the package registers its architectures)

        return MODEL_REGISTRY[arch].build_model(model_cfg, self, **kw)

    def build_criterion(self, **kw):
        from .. import criterions  # noqa: F401  (registers ctc_loss / label_smoothed_cross_entropy_v2 / transducer_loss)

        return CRITERION_REGISTRY[self.cfg.criterion_name](self, **kw)

    def build_generator(self, models, args=None, seq_gen_cls=None, extra_gen_cls_kwargs=None):
        """The decoder the reference picks per criterion (speech_recognition.py:526-596); `args` is any object with the
        generation attributes (beam, max_len_a, max_len_b, min_len, unnormalized, lenpen, unkpen, temperature,
        lm_weight, eos_factor, print_alignment, transducer_max_num_expansions_per_step, and for the attention decoder
        fairseq's search options: no_repeat_ngram_size, diverse_beam_groups, diverse_beam_strength, diversity_rate,
        sampling, sampling_topk, sampling_topp)."""
        g = lambda k, d=None: getattr(args, k, d) if args is not None else d  # noqa: E731
        extra = dict(extra_gen_cls_kwargs or {})
        if g("print_alignment", False):
            extra["print_alignment"] = True
        if self.cfg.criterion_name == "transducer_loss":
            from ..tools.transducer_greedy_decoder import TransducerGreedyDecoder

            from ..tools.transducer_beam_search_decoder import TransducerBeamSearchDecoder

            if seq_gen_cls is None:
                seq_gen_cls = TransducerGreedyDecoder if g("beam", 1) == 1 else TransducerBeamSearchDecoder
            if seq_gen_cls is TransducerBeamSearchDecoder:
                extra.update(beam_size=g("beam", 1), normalize_scores=not g("unnormalized", False),
                             expansion_beta=g("transducer_expansion_beta", 0), expansion_gamma=g("transducer_expansion_gamma", None),
                             prefix_alpha=g("transducer_prefix_alpha", None))
            return seq_gen_cls(
                models, self.target_dictionary, temperature=g("temperature", 1.0),
                max_num_expansions_per_step=g("transducer_max_num_expansions_per_step", 20),
                bos=self.target_dictionary.bos() if self.cfg.include_eos_in_transducer_loss else self.target_dictionary.eos(),
                blank=self.target_dictionary.index(self.blank_symbol),
                model_predicts_eos=self.cfg.include_eos_in_transducer_loss, **extra)
        if self.cfg.criterion_name == "ctc_loss":
            from ..tools.ctc_decoder import CTCDecoder

            # eos_factor gates eos in label-synchronous search; a CTC search has no eos step, so it does not apply
            extra.pop("eos_factor", None)
            extra.setdefault("lm_weight", g("lm_weight", 0.0))
            for k in ("word_score", "beam_size_token", "beam_threshold", "nbest", "lexicon"):
                if g(k) is not None:
                    extra.setdefault(k, g(k))
            return (seq_gen_cls or CTCDecoder)(self.target_dictionary, blank_idx=self.target_dictionary.index(self.blank_symbol),
                                               beam_size=g("beam", 1), **extra)
        from ..sequence_generator import SequenceGenerator

        # fairseq's search options and their checks (fairseq/tasks/fairseq_task.py:405-428)
        sampling, topk, topp = g("sampling", False), g("sampling_topk", -1), g("sampling_topp", -1.0)
        groups, rate = g("diverse_beam_groups", -1), g("diversity_rate", -1)
        if sum(int(c) for c in (sampling, groups > 0, g("match_source_len", False), rate > 0)) > 1:
            raise ValueError("Provided Search parameters are mutually exclusive.")
        assert topk < 0 or sampling, "--sampling-topk requires --sampling"
        assert topp < 0 or sampling, "--sampling-topp requires --sampling"
        if sampling:
            extra.update(sampling=True, sampling_topk=topk, sampling_topp=topp, sampling_seed=g("seed", 1))
        elif groups > 0:
            extra.update(diverse_beam_groups=groups, diverse_beam_strength=g("diverse_beam_strength", 0.5))
        elif g("match_source_len", False):
            pass  # the reference's LengthConstrainedBeamSearch: not supported, plain beam search as before
        elif rate > -1:
            extra.update(diversity_rate=rate)
        extra.setdefault("no_repeat_ngram_size", g("no_repeat_ngram_size", 0))
        # the decode script hands lm_model / lm_weight / eos_factor through extra_gen_cls_kwargs (speech_recognize.py:206-216);
        # stand-alone callers may leave them on `args`
        lm_weight = extra.pop("lm_weight", g("lm_weight", 0.0))
        eos_factor = extra.pop("eos_factor", g("eos_factor", None))
        return (seq_gen_cls or SequenceGenerator)(
            models, self.target_dictionary, beam_size=g("beam", 5), max_len_a=g("max_len_a", 0), max_len_b=g("max_len_b", 200),
            min_len=g("min_len", 1), normalize_scores=not g("unnormalized", False), len_penalty=g("lenpen", 1.0),
            unk_penalty=g("unkpen", 0.0), temperature=g("temperature", 1.0), lm_model=extra.pop("lm_model", None),
            lm_weight=lm_weight or 1.0, eos_factor=eos_factor, **extra)

    def build_decoder_for_validation(self, model):
        """Greedy decoders used for validation WER (speech_recognition.py:451-489)."""
        if self.cfg.criterion_name == "transducer_loss":
            from ..tools.transducer_greedy_decoder import TransducerGreedyDecoder

            self.decoder_for_validation = TransducerGreedyDecoder(
                [model], self.target_dictionary, max_num_expansions_per_step=self.cfg.max_num_expansions_per_step,
                bos=self.target_dictionary.bos() if self.cfg.include_eos_in_transducer_loss else self.target_dictionary.eos(),
                blank=self.target_dictionary.index(self.blank_symbol), model_predicts_eos=self.cfg.include_eos_in_transducer_loss)
        elif self.cfg.criterion_name == "ctc_loss":
            from ..tools.ctc_decoder import CTCDecoder

            self.decoder_for_validation = CTCDecoder(self.target_dictionary, blank_idx=self.target_dictionary.index(self.blank_symbol))
        else:
            from ..tools.simple_greedy_decoder import SimpleGreedyDecoder

            self.decoder_for_validation = SimpleGreedyDecoder([model], self.target_dictionary, for_validation=True)
        return self.decoder_for_validation

    # ---- steps ---------------------------------------------------------------------------------------------------
    def train_step(self, sample, trainer):
        """One update through espresso_b200.trainer.Trainer (fairseq/tasks/fairseq_task.py:490-522 + trainer.py:780-1097)."""
        return trainer.train_step([sample])

    def valid_step(self, sample, model, criterion):
        import torch

        model.eval()
        with torch.no_grad():
            loss, sample_size, logging_output = criterion(model, sample)
        if self.decoder_for_validation is not None:
            we, wc, ce, cc = self._inference_with_wer(self.decoder_for_validation, sample, model)
            logging_output.update(word_error=we, word_count=wc, char_error=ce, char_count=cc)
        return loss, sample_size, logging_output

    def _inference_with_wer(self, decoder, sample, model):
        tokens, _, _ = decoder.decode([model], sample)
        pred = tokens.cpu()
        target = sample["target"]
        assert pred.size(0) == target.size(0)
        d = self.target_dictionary
        ignore = set(self.extra_symbols_to_ignore)
        we = wc = ce = cc = 0
        for i in range(target.size(0)):
            if sample.get("text") is not None:
                ref_tokens = sample["text"][i]
            else:
                ref_tokens = d.string(target[i].cpu(), extra_symbols_to_ignore=ignore)
            hyp_tokens = d.string(pred[i], extra_symbols_to_ignore=ignore)
            ref_words = d.string(d.encode_line(ref_tokens, append_eos=False), bpe_symbol=self.cfg.bpe).split()
            hyp_words = d.string(d.encode_line(hyp_tokens, append_eos=False), bpe_symbol=self.cfg.bpe).split()
            e, n = edit_counts(ref_words, hyp_words)
            we, wc = we + e, wc + n
            e, n = edit_counts(list(" ".join(ref_words)), list(" ".join(hyp_words)))
            ce, cc = ce + e, cc + n
        return we, wc, ce, cc
