"""Host statement of the kernels' counter-based dropout RNG (espresso_b200/csrc/common.cuh: esp_hash_u64,
esp_dropout_keep, esp_dropout_thresh, esp_dropout_scale).

TEST INFRASTRUCTURE ONLY.  A dropout mask is a pure function of (seed, logical element index): one splitmix64-style
hash of (seed, idx >> 2) yields four 16-bit lanes, and element idx is kept iff lane idx & 3 is >= thresh(p).  Each kernel
adds the device-resident seed (ops.set_seed_tensor) to the seed of the call, modulo 2^64.  With these functions the
oracle reproduces every kernel's mask bit for bit.

All uint64 arithmetic stays in np.uint64 (mixing in Python ints would promote to float64) and wraps modulo 2^64.
"""
import numpy as np
import torch

_M64 = (1 << 64) - 1
_U = np.uint64


def combine_seed(seed, device_seed=0):
    """seed + *seed_ptr as the kernels form it (modulo 2^64)."""
    return (int(seed) + int(device_seed)) & _M64


def hash_u64(seed, g):
    """esp_hash_u64(seed, g), elementwise over g (any integer array)."""
    g = np.asarray(g).astype(np.uint64)
    with np.errstate(over="ignore"):
        z = g + _U(int(seed) & _M64) * _U(0x9E3779B97F4A7C15) + _U(0xD1B54A32D192ED03)
        z = (z ^ (z >> _U(30))) * _U(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> _U(27))) * _U(0x94D049BB133111EB)
        return z ^ (z >> _U(31))


def thresh(p):
    """esp_dropout_thresh: round(p * 65536) clamped to [0, 65535] (computed from the float32 p, in double)."""
    t = float(np.float32(p)) * 65536.0 + 0.5
    return int(min(max(t, 0.0), 65535.0))


def scale(p):
    """esp_dropout_scale: 1 / quantised keep probability, as float32 (1 for p <= 0)."""
    if not float(np.float32(p)) > 0.0:
        return 1.0
    return float(np.float32(65536.0 / (65536.0 - thresh(p))))


def keep(seed, idx, p):
    """esp_dropout_keep(seed, idx, thresh(p)) elementwise: bool array of idx's shape."""
    idx = np.asarray(idx).astype(np.uint64)
    h = hash_u64(seed, idx >> _U(2))
    lane = (h >> (_U(16) * (idx & _U(3)))) & _U(0xFFFF)
    return lane >= _U(thresh(p))


# ---- torch helpers for oracle/ops_ref.py -----------------------------------------------------------------------------
def keep_mask(seed, idx, p):
    """keep() over a torch integer tensor of logical indices -> torch.bool tensor of the same shape."""
    return torch.from_numpy(keep(seed, idx.numpy(), p))


def row_major_index(rows, cols, ld=None, row0=0):
    """Logical indices r * ld + c of a [rows, cols] block (ld defaults to cols), as int64."""
    ld = cols if ld is None else ld
    return (torch.arange(row0, row0 + rows, dtype=torch.int64)[:, None] * ld + torch.arange(cols, dtype=torch.int64)[None, :])
