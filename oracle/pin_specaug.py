"""Pin oracle/specaug.py (adaptive SpecAugment with time warping) against the REAL reference transform and cv2, and write
tests/golden/specaug_timewarp.npz.

Runs only where the reference tree and OpenCV are available (imported through oracle/refshim):
    python -m oracle.pin_specaug
(1) The oracle's statement of cv2's INTER_LINEAR rule is compared with cv2.resize over every shape a warp can ask for up
to 170 source rows.  (2) For each case, AdaptiveSpecAugmentTransform runs under fairseq's numpy_seed; the oracle must
consume the RNG the same way and agree within 1e-6.  The fixture stores, per case: the input (values that bf16 holds
exactly, so the bf16 kernel sees the same numbers), the policy, the seed, the draws and the reference output.
Cases pick a seed whose first draws give the wanted warp: W = 1, 5 and 80; w = 0 and w at both extremes; w0 at both
bounds; m = 2W + 1 and m = 2W (no warp, no warp draws); F = 83 and 40; F below freq_mask_F (no draws at all); the
Switchboard recipe's non-adaptive policy (examples/asr_swbd/run.sh) with and without a warp."""
import json
import os

import numpy as np

from oracle import refshim
from oracle import specaug as O

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
LIBRI = {"freq_mask_F": 27, "freq_mask_N": 2, "time_mask_pm": 0.04, "time_mask_ps": 0.04}
SWBD = {"freq_mask_F": 18, "time_mask_T": 70, "freq_mask_N": 2, "time_mask_N": 2, "time_mask_p": 0.2}
KEYS = ("time_warp_W", "freq_mask_N", "freq_mask_F", "time_mask_N", "time_mask_T", "time_mask_p", "time_mask_pm",
        "time_mask_ps")


def _seed_for(W, m, want):
    """The first index i whose numpy_seed(7, 1, i) stream starts with warp draws (w0, w) satisfying want(w0, w)."""
    from fairseq.data import data_utils

    for i in range(1, 1_000_000):
        with data_utils.numpy_seed(7, 1, i):
            w0 = np.random.randint(W, m - W)
            w = np.random.randint(-W + 1, W)
        if want(w0, w):
            return (7, 1, i)
    raise RuntimeError("no seed for the wanted warp")


def _cases():
    any_ = lambda w0, w: True  # noqa: E731
    c = []
    for W, m in ((1, 57), (5, 120), (80, 300)):
        c.append(("W%d_seeded" % W, dict(LIBRI, time_warp_W=W), m, 80, _seed_for(W, m, lambda w0, w: w != 0 or W == 1)))
    for W, m in ((5, 60), (80, 200)):
        c.append(("W%d_w_max" % W, dict(LIBRI, time_warp_W=W), m, 80, _seed_for(W, m, lambda w0, w: w == W - 1)))
        c.append(("W%d_w_min" % W, dict(LIBRI, time_warp_W=W), m, 80, _seed_for(W, m, lambda w0, w: w == -W + 1)))
        c.append(("W%d_w_zero" % W, dict(LIBRI, time_warp_W=W), m, 80, _seed_for(W, m, lambda w0, w: w == 0)))
        c.append(("W%d_w0_min" % W, dict(LIBRI, time_warp_W=W), m, 80, _seed_for(W, m, lambda w0, w: w0 == W and w != 0)))
        c.append(("W%d_w0_max" % W, dict(LIBRI, time_warp_W=W), m, 80,
                  _seed_for(W, m, lambda w0, w: w0 == m - W - 1 and w != 0)))
        c.append(("W%d_m_2W+1" % W, dict(LIBRI, time_warp_W=W), 2 * W + 1, 80, _seed_for(W, 2 * W + 1, lambda w0, w: w != 0)))
        c.append(("W%d_m_2W" % W, dict(LIBRI, time_warp_W=W), 2 * W, 80, (7, 1, 0)))
    c.append(("F83", dict(LIBRI, time_warp_W=5), 90, 83, _seed_for(5, 90, lambda w0, w: w != 0)))
    c.append(("F40", dict(LIBRI, time_warp_W=5), 70, 40, _seed_for(5, 70, lambda w0, w: w != 0)))
    c.append(("F_below_mask_F", dict(LIBRI, time_warp_W=5), 50, 20, (7, 1, 0)))
    c.append(("swbd", dict(SWBD, time_warp_W=0), 150, 80, (7, 1, 3)))
    c.append(("swbd_W5", dict(SWBD, time_warp_W=5), 150, 80, _seed_for(5, 150, any_)))
    return c


def pin_resize_rule():
    import cv2

    n = bad = 0
    worst = 0.0
    for S in range(2, 170):
        x = np.random.RandomState(S).randn(S, 83).astype(np.float32)
        for D in range(1, S + 80):
            a = cv2.resize(x, dsize=(83, D), interpolation=cv2.INTER_LINEAR)
            d = float(np.abs(a - O.resize_rows(x, D)).max())
            n += 1
            bad += d > 0
            worst = max(worst, d)
    print("cv2 INTER_LINEAR rule: %d resizes, %d not bit-equal, worst abs diff %.3g" % (n, bad, worst))
    assert worst <= 2.5e-7, "oracle/specaug.py does not state cv2's INTER_LINEAR rule"


def pin_cases():
    import torch
    from espresso.data.feature_transforms.adaptive_specaugment import AdaptiveSpecAugmentTransform
    from fairseq.data import data_utils

    out = {"names": np.array([])}
    names = []
    for k, (name, cfg, m, F, seed) in enumerate(_cases()):
        rs = np.random.RandomState(100 + k)
        x = torch.from_numpy(rs.randn(m, F).astype(np.float32) * 2.0 + 0.5).bfloat16().float().numpy()
        aug = AdaptiveSpecAugmentTransform.from_config_dict(cfg)
        with data_utils.numpy_seed(*seed):
            ref = aug(x)
            after_ref = np.random.randint(0, 2**31 - 1)
        full = {kk: cfg.get(kk, O.adaptive_specaugment.__defaults__[KEYS.index(kk)]) for kk in KEYS}
        with data_utils.numpy_seed(*seed):
            got, warp, fm, tm = O.adaptive_specaugment(x, **full)
            after_oracle = np.random.randint(0, 2**31 - 1)
        d = float(np.abs(got - ref).max())
        print("%-16s m=%3d F=%d seed=%s warp=%s masks f=%s t=%d |oracle - reference|=%.3g" % (
            name, m, F, seed, warp, fm, len(tm), d))
        assert after_ref == after_oracle, "the oracle consumes the RNG differently (%s)" % name
        assert d <= 1e-6, "oracle disagrees with the reference (%s)" % name
        names.append(name)
        out["x_%d" % k] = x
        out["out_%d" % k] = np.asarray(ref, dtype=np.float32)
        out["cfg_%d" % k] = np.array(json.dumps(cfg))
        out["seed_%d" % k] = np.array(seed, dtype=np.int64)
        out["warp_%d" % k] = np.array(warp if warp is not None else [], dtype=np.int32).reshape(-1, 2)
        out["fm_%d" % k] = np.array(fm, dtype=np.int32).reshape(-1, 2)
        out["tm_%d" % k] = np.array(tm, dtype=np.int32).reshape(-1, 2)
    out["names"] = np.array(names)
    np.savez_compressed(os.path.join(GOLDEN, "specaug_timewarp.npz"), **out)
    print("%d cases -> tests/golden/specaug_timewarp.npz" % len(names))


if __name__ == "__main__":
    refshim.activate()
    pin_resize_rule()
    pin_cases()
