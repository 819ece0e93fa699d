"""Mini-batch assembly with the reference's layout (host logic; espresso/data/asr_dataset.py:17-136,
espresso/tools/utils.py:97-113 `collate_frames`, fairseq/data/data_utils.py:36-90 `collate_tokens`).

collate(samples, pad_idx, eos_idx) -> {"id", "utt_id", "nsentences", "ntokens",
    "net_input": {"src_tokens" f32 [B, Tmax, F] (or raw waveforms f32 [B, Nmax], or for FLAC items a PackedFlac that
                  espresso_b200.data.flac.to_device decodes into them), "src_lengths" i32 [B],
                  "prev_output_tokens" i64 [B, Umax]}, "target" i64 [B, Umax], "text"}
Rows are sorted by source length, longest first (stable for ties); features are right-padded with 0.0, token rows with
pad_idx; prev_output_tokens is the target with its eos moved to the front (input feeding), or `maybe_bos_idx` prepended.
Only right padding is implemented: it is what the ASR task uses (left_pad_source = left_pad_target = False).

In training the samples carry the host-drawn SpecAugment descriptors ("freq_masks", "time_masks" and, for a policy
with time warping, "time_warp" from espresso_b200.data.specaugment); they are packed into the `freq_masks` / `time_masks`
tensors and the int32 [B, 2] `time_warp` tensor that esp_frontend_fbank and esp_specaug_features consume, for raw
waveforms ("source" 1-D) and features alike."""
import numpy as np
import torch

from . import flac as _flac, specaugment as _SA


def collate_frames(values, pad_value=0.0, pad_to_multiple=1):
    """List of [T_i, F] (or 1-D [N_i]) float tensors -> right-padded [B, Tmax, F] ([B, Nmax])."""
    size = max(v.size(0) for v in values)
    if pad_to_multiple > 1:
        size = (size + pad_to_multiple - 1) // pad_to_multiple * pad_to_multiple
    shape = (len(values), size) + tuple(values[0].shape[1:])
    out = values[0].new_full(shape, pad_value)
    for i, v in enumerate(values):
        out[i, : v.size(0)] = v
    return out


def collate_tokens(values, pad_idx, eos_idx=None, move_eos_to_beginning=False, pad_to_multiple=1):
    """List of 1-D int64 token tensors -> right-padded [B, Umax]; optionally rotate the trailing eos to position 0."""
    size = max(v.size(0) for v in values)
    if pad_to_multiple > 1:
        size = (size + pad_to_multiple - 1) // pad_to_multiple * pad_to_multiple
    out = values[0].new_full((len(values), size), pad_idx)
    for i, v in enumerate(values):
        n = v.size(0)
        if move_eos_to_beginning:
            out[i, 0] = v[-1] if eos_idx is None else eos_idx
            out[i, 1:n] = v[:-1]
        else:
            out[i, :n] = v
    return out


def collate(samples, pad_idx, eos_idx, left_pad_source=False, left_pad_target=False, input_feeding=True, maybe_bos_idx=None,
            pad_to_multiple=1):
    if len(samples) == 0:
        return {}
    if left_pad_source or left_pad_target:
        raise NotImplementedError("the ASR path pads on the right (asr_dataset.py: left_pad_* default False in the task)")
    is_flac = [isinstance(s["source"], _flac.FlacStream) for s in samples]
    if any(is_flac) and not all(is_flac):
        raise ValueError("a batch mixes FLAC and decoded (WAVE) audio: give a manifest's utterances one format")
    lengths = np.array([s["source"].total_samples if f else s["source"].size(0) for s, f in zip(samples, is_flac)],
                       dtype=np.int64)
    order = np.argsort(-lengths, kind="mergesort")  # longest first, stable
    pick = lambda xs: [xs[i] for i in order]  # noqa: E731
    if is_flac[0]:  # compressed: decoded on the device by espresso_b200.data.flac.to_device
        src = _flac.pack(pick([s["source"] for s in samples]), names=pick([s.get("utt_id") for s in samples]),
                         pad_to_multiple=pad_to_multiple)
    else:
        src = collate_frames(pick([s["source"] for s in samples]), 0.0, pad_to_multiple)
    batch = {
        "id": torch.tensor(pick([int(s["id"]) for s in samples]), dtype=torch.long),
        "utt_id": pick([s.get("utt_id") for s in samples]),
        "nsentences": len(samples),
        "net_input": {"src_tokens": src, "src_lengths": torch.tensor(lengths[order], dtype=torch.int32)},
        "target": None,
        "text": pick([s["text"] for s in samples]) if samples[0].get("text") is not None else None,
    }
    if samples[0].get("target") is not None:
        tg = pick([s["target"] for s in samples])
        batch["target"] = collate_tokens(tg, pad_idx, pad_to_multiple=pad_to_multiple)
        batch["ntokens"] = int(sum(int((t != pad_idx).sum()) for t in tg))
        if samples[0].get("prev_output_tokens") is not None:
            batch["net_input"]["prev_output_tokens"] = collate_tokens(pick([s["prev_output_tokens"] for s in samples]), pad_idx)
        elif input_feeding:
            prev = collate_tokens(tg, pad_idx, eos_idx, move_eos_to_beginning=(maybe_bos_idx is None),
                                  pad_to_multiple=pad_to_multiple)
            if maybe_bos_idx is not None:
                prev = torch.cat([prev.new_full((len(samples), 1), maybe_bos_idx), prev], dim=1)
            batch["net_input"]["prev_output_tokens"] = prev
    else:
        batch["ntokens"] = int(lengths.sum())
    if samples[0].get("freq_masks") is not None:  # on-device front end: pack the host-drawn SpecAugment descriptors
        fm, tm = _SA.pack_masks(pick([s["freq_masks"] for s in samples]), pick([s["time_masks"] for s in samples]))
        batch["net_input"]["freq_masks"] = torch.from_numpy(fm)
        batch["net_input"]["time_masks"] = torch.from_numpy(tm)
    if "time_warp" in samples[0]:
        batch["net_input"]["time_warp"] = torch.from_numpy(_SA.pack_warps(pick([s["time_warp"] for s in samples])))
    return batch
