"""Datasets of the `speech_recognition_espresso` task (host side): the JSON manifest, the audio / feature dataset, the
transcript dataset and their pairing (espresso/tasks/speech_recognition.py:127-269, espresso/data/feat_text_dataset.py:35-161,
333-396, espresso/data/asr_dataset.py:139-411).

native difference: for "wave" / "command" entries the item is the RAW waveform (float32, int16 scale) plus, in training, the
SpecAugment mask descriptors drawn on the host with the reference's RNG protocol (numpy_seed(seed, epoch, index),
feat_text_dataset.py:151-153); fbank + CMVN + masking run on the device for the whole batch (csrc/frontend.cu) instead of per
utterance in DataLoader workers.  "feat" entries (Kaldi archives) are read as matrices exactly like the reference."""
import itertools
import json
import os
import re
from collections import OrderedDict
from io import BytesIO
from subprocess import PIPE, run

import numpy as np
import torch

from . import batching, flac as _flac, specaugment as SA
from .audio_io import get_waveform, num_frames_of, read_kaldi_mat
from .collate import collate


class AudioFeatDataset(torch.utils.data.Dataset):
    def __init__(self, utt_ids, rxfiles, utt2num_frames=None, feat_dim=None, feature_type=None, seed=1, specaugment_config=None,
                 frame_length_ms=25.0, frame_shift_ms=10.0):
        assert len(utt_ids) == len(rxfiles)
        self.utt_ids, self.rxfiles, self.size = list(utt_ids), list(rxfiles), len(utt_ids)
        first = self.rxfiles[0].strip()
        if re.search(r"\.ark:\d+$", first):
            self.input_format = "feat"
            self.feat_dim = read_kaldi_mat(first).shape[1]
        else:
            self.input_format = "command" if first.endswith("|") else "wave"
            self.feat_dim, self.feature_type = feat_dim, feature_type
            if feat_dim is None or feature_type != "fbank":
                raise ValueError("waveform input needs feat_dim and feature_type='fbank' (the on-device front end)")
        self.frame_length_ms, self.frame_shift_ms = frame_length_ms, frame_shift_ms
        if utt2num_frames is not None and len(utt2num_frames) > 0:
            assert len(utt2num_frames) == self.size
            sizes = utt2num_frames
        else:
            sizes = [self._count_frames(r) for r in self.rxfiles]
        self.sizes = np.asarray(sizes, dtype=np.int32)
        self.specaug = SA.AdaptiveSpecAugmentConfig.from_config_dict(specaugment_config) if specaugment_config else None
        self.seed, self.epoch = seed, 1

    def _open(self, rx):
        return BytesIO(run(rx.strip()[:-1], shell=True, stdout=PIPE).stdout) if self.input_format == "command" else rx

    def _read_audio(self, rx):
        """float32 waveform in int16 range, or for FLAC (a .flac path, or command output starting with fLaC) the
        compressed stream, decoded later on the device for the whole batch (espresso_b200.data.flac.to_device)."""
        if self.input_format == "command":
            buf = run(rx.strip()[:-1], shell=True, stdout=PIPE).stdout
            if _flac.is_flac(buf):
                return _flac.read_stream(buf)
            rx = BytesIO(buf)
        elif rx.strip().lower().endswith(".flac"):
            with open(rx.strip(), "rb") as f:
                return _flac.read_stream(f.read())
        wav, _ = get_waveform(rx, normalization=False, always_2d=False)
        return torch.from_numpy(wav)

    def _count_frames(self, rx):
        return num_frames_of(self._open(rx) if self.input_format != "feat" else rx, self.frame_length_ms, self.frame_shift_ms)

    def set_epoch(self, epoch):
        self.epoch = epoch

    def filter_and_reorder(self, indices):
        indices = np.asarray(indices)
        assert len(np.unique(indices)) == len(indices), "Duplicate elements in indices."
        self.utt_ids = [self.utt_ids[i] for i in indices]
        self.rxfiles = [self.rxfiles[i] for i in indices]
        self.sizes = self.sizes[indices]
        self.size = len(self.utt_ids)

    def __len__(self):
        return self.size

    def __getitem__(self, i):
        """-> dict(source = float32 [frames, dim] features, [samples] waveform or a FlacStream, freq_masks / time_masks or
        None), and time_warp (None or (w0, w)) when the SpecAugment policy warps time (time_warp_W > 0)."""
        if i < 0 or i >= self.size:
            raise IndexError("index out of range")
        if self.input_format == "feat":
            src = torch.from_numpy(read_kaldi_mat(self.rxfiles[i])).float()
            frames = src.size(0)
        else:
            src = self._read_audio(self.rxfiles[i])
            frames = int(self.sizes[i])
        fm = tm = None
        if self.specaug is not None and self.specaug.time_warp_W > 0:
            with SA.numpy_seed(self.seed, self.epoch, i):
                warp, fm, tm = SA.draw_specaugment(self.specaug, frames, self.feat_dim)
            return {"source": src, "freq_masks": fm, "time_masks": tm, "time_warp": warp}
        if self.specaug is not None:
            with SA.numpy_seed(self.seed, self.epoch, i):
                fm, tm = SA.draw_masks(self.specaug, frames, self.feat_dim)
        return {"source": src, "freq_masks": fm, "time_masks": tm}


class AsrTextDataset(torch.utils.data.Dataset):
    """Transcripts: kept as text, tokenised on access through the dictionary's word-piece encoder."""

    def __init__(self, utt_ids, texts, dictionary=None, append_eos=True):
        assert len(utt_ids) == len(texts)
        self.utt_ids, self.texts, self.dictionary, self.append_eos = list(utt_ids), list(texts), dictionary, append_eos
        self.size = len(self.utt_ids)
        enc = dictionary.wordpiece_encode if dictionary is not None else (lambda t: t)
        extra = 1 if (append_eos and dictionary is not None) else 0
        self.sizes = np.asarray([len(enc(t).split()) + extra for t in texts], dtype=np.int32)

    def filter_and_reorder(self, indices):
        indices = np.asarray(indices)
        self.utt_ids = [self.utt_ids[i] for i in indices]
        self.texts = [self.texts[i] for i in indices]
        self.sizes = self.sizes[indices]
        self.size = len(self.utt_ids)

    def __len__(self):
        return self.size

    def __getitem__(self, i):
        if i < 0 or i >= self.size:
            raise IndexError("index out of range")
        if self.dictionary is None:
            return None, self.texts[i]
        ids = self.dictionary.encode_line(self.dictionary.wordpiece_encode(self.texts[i]), add_if_not_exist=False,
                                          append_eos=self.append_eos).long()
        return ids, self.texts[i]


class AsrDataset(torch.utils.data.Dataset):
    """Pairs audio with transcripts by utterance id (asr_dataset.py:213-243: utterances missing on either side are dropped,
    the text side is re-ordered to the audio side) and assembles mini-batches."""

    def __init__(self, src, src_sizes, tgt=None, tgt_sizes=None, dictionary=None, shuffle=True, input_feeding=True,
                 prepend_bos_as_input_feeding=False, pad_to_multiple=1, batch_based_on_both_src_tgt=False, seed=1):
        self.src, self.tgt, self.dictionary = src, tgt, dictionary
        self.shuffle, self.input_feeding, self.pad_to_multiple = shuffle, input_feeding, pad_to_multiple
        self.prepend_bos = prepend_bos_as_input_feeding
        self.both, self.seed, self.epoch = batch_based_on_both_src_tgt, seed, 1
        if tgt is not None:
            self._match()
        self.src_sizes = np.asarray(self.src.sizes)
        self.tgt_sizes = np.asarray(self.tgt.sizes) if self.tgt is not None else None

    def _match(self):
        tgt_pos = {u: i for i, u in enumerate(self.tgt.utt_ids)}
        keep_src = [i for i, u in enumerate(self.src.utt_ids) if u in tgt_pos]
        if len(keep_src) == 0:
            raise ValueError("audio and text share no utterance id")
        self.src.filter_and_reorder(keep_src)
        self.tgt.filter_and_reorder([tgt_pos[u] for u in self.src.utt_ids])
        assert self.src.utt_ids == self.tgt.utt_ids

    def set_epoch(self, epoch):
        self.epoch = epoch
        self.src.set_epoch(epoch)

    def __len__(self):
        return len(self.src)

    def num_tokens(self, i):
        """Frames (plus target tokens when batching on both sides), asr_dataset.py:331-340."""
        n = int(self.src_sizes[i])
        return n + int(self.tgt_sizes[i]) if (self.both and self.tgt_sizes is not None) else n

    def size(self, i):
        return int(self.src_sizes[i]), int(self.tgt_sizes[i]) if self.tgt_sizes is not None else 0

    def __getitem__(self, i):
        item = dict(self.src[i])
        ids, text = self.tgt[i] if self.tgt is not None else (None, None)
        item.update(id=i, utt_id=self.src.utt_ids[i], target=ids, text=text)
        return item

    def collater(self, samples):
        d = self.dictionary
        bos = d.bos() if (self.prepend_bos and d is not None) else None
        return collate(samples, pad_idx=d.pad() if d is not None else 0, eos_idx=d.eos() if d is not None else 0,
                       input_feeding=self.input_feeding, maybe_bos_idx=bos, pad_to_multiple=self.pad_to_multiple)

    def ordered_indices(self):
        """Random order then stable sorts by target and source length (asr_dataset.py:342-371), seeded per epoch."""
        seed = (self.seed + self.epoch) if self.shuffle else None
        return batching.ordered_indices(self.src_sizes, self.tgt_sizes, shuffle_seed=seed)

    def batch_by_size(self, indices, max_tokens=None, max_sentences=None, required_batch_size_multiple=1):
        ntok = self.src_sizes.astype(np.int64) + (self.tgt_sizes if (self.both and self.tgt_sizes is not None) else 0)
        return batching.batch_by_size(indices, ntok, max_tokens, max_sentences, required_batch_size_multiple)


def get_asr_dataset_from_json(data_path, split, tgt_dict, combine=False, upsample_primary=1, shuffle=True, pad_to_multiple=1,
                              autoregressive=True, prepend_bos_as_input_feeding=False, is_training_set=False,
                              batch_based_on_both_src_tgt=False, seed=1, specaugment_config=None):
    """The manifest of espresso/tools/asr_prep_json.py: {utt_id: {"feat" | "wave" | "command": ..., "text": ...,
    "utt2num_frames": ...}}; `split`, `split1`, ... are concatenated when combine is set
    (speech_recognition.py:127-269)."""
    srcs, tgts = [], []
    for k in itertools.count():
        path = os.path.join(data_path, "%s%s.json" % (split, str(k) if k > 0 else ""))
        if not os.path.isfile(path):
            if k > 0:
                break
            raise FileNotFoundError("Dataset not found: %s" % path)
        with open(path, "rb") as f:
            loaded = json.load(f, object_pairs_hook=OrderedDict)
        utt_ids, audios, texts, nframes = [], [], [], []
        for utt_id, val in loaded.items():
            key = next((k_ for k_ in ("feat", "wave", "command") if k_ in val), None)
            if key is None:
                raise KeyError("'feat', 'wave' or 'command' should be present as a field for the entry %s in %s" % (utt_id, path))
            utt_ids.append(utt_id)
            audios.append(val[key])
            if "text" in val:
                texts.append(val["text"])
            if "utt2num_frames" in val:
                nframes.append(int(val["utt2num_frames"]))
        assert len(nframes) == 0 or len(nframes) == len(utt_ids)
        kw = {} if "feat" in next(iter(loaded.values())) else {"feat_dim": 80, "feature_type": "fbank"}
        if specaugment_config is not None and is_training_set:
            kw["specaugment_config"] = eval(specaugment_config) if isinstance(specaugment_config, str) else specaugment_config
        srcs.append(AudioFeatDataset(utt_ids, audios, utt2num_frames=nframes, seed=seed, **kw))
        if texts:
            assert len(texts) == len(utt_ids) and tgt_dict is not None
            tgts.append(AsrTextDataset(utt_ids, texts, tgt_dict, append_eos=autoregressive))
        if not combine:
            break
    assert len(tgts) in (0, len(srcs))
    if len(srcs) > 1:
        if any(s.feat_dim != srcs[0].feat_dim or s.input_format != srcs[0].input_format for s in srcs):
            raise ValueError("feature dimension / input format does not match across multiple json files")
        ratios = [upsample_primary] + [1] * (len(srcs) - 1)
        src, tgt = _concat(srcs, ratios), (_concat(tgts, ratios) if tgts else None)
    else:
        src, tgt = srcs[0], (tgts[0] if tgts else None)
    return AsrDataset(src, src.sizes, tgt, tgt.sizes if tgt is not None else None, tgt_dict, shuffle=shuffle,
                      input_feeding=autoregressive, prepend_bos_as_input_feeding=prepend_bos_as_input_feeding,
                      pad_to_multiple=pad_to_multiple, batch_based_on_both_src_tgt=batch_based_on_both_src_tgt, seed=seed)


def _concat(parts, ratios):
    """ConcatDataset with integer up-sampling of the first part (fairseq/data/concat_dataset.py), flattened into the first
    dataset object: items are cheap references (paths / strings), so repeating them costs nothing."""
    field = "rxfiles" if hasattr(parts[0], "rxfiles") else "texts"
    ids, items, sizes = [], [], []
    for p, r in zip(parts, ratios):
        for _ in range(r):
            ids += p.utt_ids
            items += getattr(p, field)
            sizes.append(p.sizes)
    first = parts[0]
    first.utt_ids, first.sizes, first.size = ids, np.concatenate(sizes), len(ids)
    setattr(first, field, items)
    return first
