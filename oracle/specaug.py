"""Oracle: adaptive SpecAugment WITH time warping (numpy), and the per-op reference of `ops.specaug_features` (torch).

Restates espresso/data/feature_transforms/adaptive_specaugment.py:77-136, including the warp of :94-109, which calls
cv2.resize(part, dsize=(num_freqs, rows), interpolation=cv2.INTER_LINEAR) on the two parts of the time axis.  The
OpenCV wheels for x86-64 hand a float32 INTER_LINEAR resize to Intel IPP (cv2.getBuildInformation(): "Custom HAL: YES
(ipp)"), and its rule, for output index r of an axis of S source samples resized to D, is:
    f = (r + 0.5) * (1 / ((double)D / S)) - 0.5;  sy = floor(f);  fy = float32(f - sy)     (coordinate in double)
    sy < 0       -> sy = 0,     fy = 0
    sy >= S - 1  -> sy = S - 1, fy = 0
    out[r] = fma(in[sy + 1] - in[sy], fy, in[sy])                     (float32 difference, one rounding for the fma)
OpenCV's own fallback (resizeGeneric_) rounds the coordinate to float32 before it takes floor and fraction, which moves
fy by up to r * 2^-24.  oracle/pin_specaug.py compares the rule above with cv2: over every S in [2, 170) and D in
[1, S + 80), 26,442 of 27,636 resizes of unit-variance data are equal bit for bit, and the others differ by at most
2.4e-7 (2 ulp) in some elements.
The frequency axis keeps its size (scale 1, fy = 0 everywhere): a copy.  oracle/pin_specaug.py checks this rule against
cv2 itself and the real reference transform before it writes tests/golden/specaug_timewarp.npz.
Test infrastructure only (see oracle/__init__.py).
"""
import math

import numpy as np
import torch


def linear_rows(S, D):
    """cv2 INTER_LINEAR source rows and weight for resizing S rows to D: (sy0 [D], sy1 [D], fy float32 [D])."""
    scale = 1.0 / (float(D) / float(S))
    sy0 = np.zeros(D, np.int64)
    fy = np.zeros(D, np.float32)
    for r in range(D):
        f = (r + 0.5) * scale - 0.5
        sy = math.floor(f)
        f = np.float32(f - sy)
        if sy < 0:
            sy, f = 0, np.float32(0)
        if sy >= S - 1:
            sy, f = S - 1, np.float32(0)
        sy0[r], fy[r] = sy, f
    return sy0, np.minimum(sy0 + 1, S - 1), fy


def resize_rows(x, D):
    """cv2.resize(x, dsize=(x.shape[1], D), interpolation=cv2.INTER_LINEAR) for float32 x [S, F]."""
    x = np.asarray(x, np.float32)
    sy0, sy1, fy = linear_rows(x.shape[0], D)
    a, d = x[sy0], x[sy1] - x[sy0]  # float32 difference
    return (a.astype(np.float64) + d.astype(np.float64) * fy[:, None].astype(np.float64)).astype(np.float32)  # = fma


def warp_frames(x, w0, w):
    """adaptive_specaugment.py:100-109: frames [0, w0) -> w0 + w rows, [w0, m) -> m - w0 - w rows."""
    m = x.shape[0]
    return np.concatenate([resize_rows(x[:w0], w0 + w), resize_rows(x[w0:], m - w0 - w)], axis=0)


def adaptive_specaugment(spec, time_warp_W=0, freq_mask_N=0, freq_mask_F=0, time_mask_N=0, time_mask_T=0,
                         time_mask_p=0.0, time_mask_pm=None, time_mask_ps=None):
    """adaptive_specaugment.py:77-136 (mask_value None: the local mean) on float32 spec [m, F]; draws from the global
    NumPy RNG.  Returns (out, warp or None, [(f0, f)], [(t0, t)])."""
    out = spec.copy()
    m, nf = spec.shape
    fill = spec.mean()  # before the warp
    warp, fmasks, tmasks = None, [], []
    if m == 0 or nf < freq_mask_F:
        return out, warp, fmasks, tmasks
    if time_warp_W > 0 and 2 * time_warp_W < m:
        w0 = np.random.randint(time_warp_W, m - time_warp_W)
        w = np.random.randint(-time_warp_W + 1, time_warp_W)
        out = warp_frames(out, w0, w)
        warp = (int(w0), int(w))
    for _ in range(freq_mask_N):
        f = np.random.randint(0, freq_mask_F)
        f0 = np.random.randint(0, nf - f)
        fmasks.append((int(f0), int(f)))
        if f != 0:
            out[:, f0:f0 + f] = fill
    max_t = min(time_mask_T, math.floor(m * time_mask_p)) if time_mask_ps is None else math.floor(m * time_mask_ps)
    if max_t < 1:
        return out, warp, fmasks, tmasks
    n = time_mask_N if time_mask_pm is None else min(20, math.floor(m * time_mask_pm))
    for _ in range(n):
        t = np.random.randint(0, max_t)
        t0 = np.random.randint(0, m - t)
        tmasks.append((int(t0), int(t)))
        if t != 0:
            out[t0:t0 + t, :] = fill
    return out, warp, fmasks, tmasks


def specaug_features(x, lens, time_warp=None, freq_masks=None, time_masks=None, out_dtype=None):
    """Per-op reference of ops.specaug_features (same signature, CPU tensors): float32 warp with the cv2 rule, fill =
    float32 of the float64 mean of the m x F input values before the warp, frames >= m zero."""
    B, T, F = x.shape
    out_dtype = x.dtype if out_dtype is None else out_dtype
    out = torch.zeros(B, T, F, dtype=torch.float32)
    xs = x.float().numpy()
    for b in range(B):
        m = min(max(int(lens[b]), 0), T)
        if m == 0:
            continue
        y = xs[b, :m].copy()
        if time_warp is not None:
            w0, w = (int(v) for v in time_warp[b])
            if w != 0 and 0 < w0 < m and 0 < w0 + w < m:
                y = warp_frames(y, w0, w)
        fill = np.float32(xs[b, :m].astype(np.float64).mean())
        if freq_masks is not None:
            for f0, f in freq_masks[b].tolist():
                if f > 0:
                    y[:, f0:f0 + f] = fill
        if time_masks is not None:
            for t0, t in time_masks[b].tolist():
                if t > 0:
                    y[t0:t0 + t, :] = fill
        out[b, :m] = torch.from_numpy(y)
    return out.to(out_dtype)
