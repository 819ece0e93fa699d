"""Host side of the fused front end: draw SpecAugment mask descriptors with the reference's RNG.

The reference applies ``AdaptiveSpecAugmentTransform`` per utterance on the CPU under
``numpy_seed(seed, epoch, index)`` (espresso/data/feat_text_dataset.py:151-153,
fairseq/data/data_utils.py:127-140).  The native path keeps exactly those NumPy draws on the host -- same
order, same bounds (espresso/data/feature_transforms/adaptive_specaugment.py:94-134) -- and uploads only
the descriptors: the time warp (w0, w) and the (start, width) masks.  The device kernels warp the time axis and paint the
masks with the utterance mean.
"""
import contextlib
import math
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np

MAX_TIME_MASKS = 20  # adaptive policy cap: min(20, floor(m * pm))  (adaptive_specaugment.py:124-129)


@contextlib.contextmanager
def numpy_seed(seed, *addl_seeds):
    """Same contract as fairseq.data.data_utils.numpy_seed (data_utils.py:127-140)."""
    if seed is None:
        yield
        return
    if len(addl_seeds) > 0:
        seed = int(hash((seed, *addl_seeds)) % 1e6)
    state = np.random.get_state()
    np.random.seed(seed)
    try:
        yield
    finally:
        np.random.set_state(state)


@dataclass
class AdaptiveSpecAugmentConfig:
    """Mirror of the transform's config keys (adaptive_specaugment.py:20-45; specaugment.py:20-45)."""
    time_warp_W: int = 0
    freq_mask_N: int = 0
    freq_mask_F: int = 0
    time_mask_N: int = 0
    time_mask_T: int = 0
    time_mask_p: float = 0.0
    time_mask_pm: Optional[float] = None
    time_mask_ps: Optional[float] = None

    @classmethod
    def from_config_dict(cls, config=None):
        c = {} if config is None else dict(config)
        cfg = cls(**{k: c[k] for k in c if k in cls.__dataclass_fields__})
        if cfg.time_warp_W < 0:
            raise ValueError("time_warp_W must be >= 0, got %d" % cfg.time_warp_W)
        return cfg


# time_warp descriptor of an utterance without a warp draw.  Any (w0, 0) leaves the features unchanged.
NO_WARP = (0, 0)


def draw_specaugment(cfg: AdaptiveSpecAugmentConfig, num_frames: int, num_freqs: int = 80
                     ) -> Tuple[Optional[Tuple[int, int]], List[Tuple[int, int]], List[Tuple[int, int]]]:
    """Consume the global NumPy RNG exactly like AdaptiveSpecAugmentTransform.__call__ and return
    (warp, [(f0, f)], [(t0, t)]).  warp = (w0, w) when a time warp was drawn (the first w0 frames are resized to w0 + w,
    the other m - w0 to m - w0 - w), else None."""
    warp, fmasks, tmasks = None, [], []
    if num_frames == 0 or num_freqs < cfg.freq_mask_F:
        return warp, fmasks, tmasks
    W = cfg.time_warp_W
    if W > 0 and 2 * W < num_frames:
        w0 = np.random.randint(W, num_frames - W)
        w = np.random.randint(-W + 1, W)
        warp = (int(w0), int(w))
    fmasks, tmasks = _draw_mask_lists(cfg, num_frames, num_freqs)
    return warp, fmasks, tmasks


def draw_masks(cfg: AdaptiveSpecAugmentConfig, num_frames: int, num_freqs: int = 80
               ) -> Tuple[List[Tuple[int, int]], List[Tuple[int, int]]]:
    """Consume the global NumPy RNG exactly like AdaptiveSpecAugmentTransform.__call__ with time_warp_W = 0 and return
    ([(f0, f)], [(t0, t)]).  A policy with a time warp draws through `draw_specaugment`."""
    if cfg.time_warp_W != 0:
        raise ValueError("draw_masks skips the time-warp draws; use draw_specaugment for time_warp_W = %d"
                         % cfg.time_warp_W)
    if num_frames == 0 or num_freqs < cfg.freq_mask_F:
        return [], []
    return _draw_mask_lists(cfg, num_frames, num_freqs)


def _draw_mask_lists(cfg, num_frames, num_freqs):
    fmasks, tmasks = [], []
    for _ in range(cfg.freq_mask_N):
        f = np.random.randint(0, cfg.freq_mask_F)
        f0 = np.random.randint(0, num_freqs - f)
        fmasks.append((int(f0), int(f)))
    if cfg.time_mask_ps is None:
        max_t = min(cfg.time_mask_T, math.floor(num_frames * cfg.time_mask_p))
    else:
        max_t = math.floor(num_frames * cfg.time_mask_ps)
    if max_t < 1:
        return fmasks, tmasks
    n = cfg.time_mask_N if cfg.time_mask_pm is None else min(MAX_TIME_MASKS, math.floor(num_frames * cfg.time_mask_pm))
    for _ in range(n):
        t = np.random.randint(0, max_t)
        t0 = np.random.randint(0, num_frames - t)
        tmasks.append((int(t0), int(t)))
    return fmasks, tmasks


def pack_masks(per_utt_f, per_utt_t):
    """Pad per-utterance descriptor lists into int32 arrays [B, NF, 2] and [B, NT, 2] (width 0 = no-op)."""
    B = len(per_utt_f)
    nf = max([len(x) for x in per_utt_f] + [1])
    nt = max([len(x) for x in per_utt_t] + [1])
    fm = np.zeros((B, nf, 2), dtype=np.int32)
    tm = np.zeros((B, nt, 2), dtype=np.int32)
    for b in range(B):
        for i, (a, w) in enumerate(per_utt_f[b]):
            fm[b, i] = (a, w)
        for i, (a, w) in enumerate(per_utt_t[b]):
            tm[b, i] = (a, w)
    return fm, tm


def pack_warps(per_utt_warp):
    """Per-utterance warp draws (None or (w0, w)) -> int32 [B, 2], NO_WARP where none was drawn."""
    return np.array([NO_WARP if w is None else w for w in per_utt_warp], dtype=np.int32).reshape(-1, 2)
