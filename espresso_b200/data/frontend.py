"""On-device feature front end: the native replacement of `AudioFeatDataset._get_features`
(espresso/data/feat_text_dataset.py:128-161).  The dataset side only has to yield raw waveforms (int16
range, like fairseq/data/audio/audio_utils.py:117-118) and draw SpecAugment descriptors
(espresso_b200/data/specaugment.py); everything else is one kernel launch per batch."""
import numpy as np
import torch

from .. import ops as _ops


class OnTheFlyFbank:
    def __init__(self, cmvn_mean=None, cmvn_std=None, out_dtype=torch.bfloat16):
        """cmvn_mean / cmvn_std: float64 arrays [80] as stored by compute_global_cmvn_stats.py (`.npz`), or None."""
        self.out_dtype = out_dtype
        self._mean_np = None if cmvn_mean is None else np.asarray(cmvn_mean, dtype=np.float64)
        self._std_np = None if cmvn_std is None else np.asarray(cmvn_std, dtype=np.float64)
        self._dev = {}
        self._ws = {}

    @classmethod
    def from_npz(cls, path, **kw):
        st = np.load(path)
        return cls(st["mean"], st["std"], **kw)  # keys of global_cmvn.py:20-22

    def _stats(self, device):
        if self._mean_np is None:
            return None, None
        k = str(device)
        if k not in self._dev:
            self._dev[k] = (torch.from_numpy(self._mean_np.astype(np.float32)).to(device),
                            torch.from_numpy(self._std_np.astype(np.float32)).to(device))
        return self._dev[k]

    def __call__(self, wave, n_samples, freq_masks=None, time_masks=None, time_warp=None):
        """time_warp int32 [B, 2] or None.  Without it, masks are painted inside the fused front end (one call).  With it,
        the front end writes fp32 features and esp_specaug_features warps and masks them (fill: the mean before the
        warp, as the reference takes it)."""
        mean, std = self._stats(wave.device)
        B = wave.shape[0]
        k = (str(wave.device), B)
        if k not in self._ws:  # zero once; the kernel leaves its workspace clean
            self._ws[k] = torch.zeros(max(B, 1) * 16, dtype=torch.uint8, device=wave.device)
        if time_warp is None:
            return _ops.frontend_fbank(wave, n_samples.to(torch.int32), mean, std, freq_masks, time_masks,
                                       out_dtype=self.out_dtype, workspace=self._ws[k])
        feats, lens = _ops.frontend_fbank(wave, n_samples.to(torch.int32), mean, std, out_dtype=torch.float32,
                                          workspace=self._ws[k])
        return _ops.specaug_features(feats, lens, time_warp, freq_masks, time_masks, out_dtype=self.out_dtype), lens
