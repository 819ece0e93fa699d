"""CPU: the host statement of the kernels' counter-based dropout RNG (oracle/dropout_rng.py) against known answers.

The values below were produced by a host build of esp_hash_u64 / esp_dropout_keep / esp_dropout_thresh /
esp_dropout_scale from espresso_b200/csrc/common.cuh; they pin the oracle's numpy statement bit for bit, so every
kernel test and the engine-versus-oracle tests that rely on it compare against the kernels' own convention."""
import numpy as np
import pytest
import torch

from oracle import dropout_rng as R

# (seed, idx, p, esp_hash_u64(seed, idx >> 2), esp_dropout_keep(seed, idx, esp_dropout_thresh(p)))
KNOWN = [
    (0, 0, 1e-6, 0x8209B480FAED1B10, 1),
    (0, 2, 0.25, 0x8209B480FAED1B10, 1),
    (0, 4, 0.9999, 0x8B2FAAB3724AC25B, 0),
    (0, 123456789, 0.1, 0xD4E149DB7EF4D3C9, 1),
    (1, 1, 0.1, 0x2D0F28C7E7E786B2, 1),
    (1, 3, 0.5, 0x2D0F28C7E7E786B2, 0),
    (1, 1001, 1e-6, 0x57E8C24A96B13BB1, 1),
    (1, 1099511627782, 0.25, 0x711C63B971331D4D, 1),
    (12345, 2, 0.25, 0x1A620B1863A763BC, 0),
    (12345, 4, 0.9999, 0x3CAED3C992B1D988, 0),
    (12345, 123456789, 0.1, 0x9FA50661C349FCF6, 1),
    (12345, 0, 0.5, 0x1A620B1863A763BC, 0),
    (9223372036854775807, 3, 0.5, 0x8BA00A5C98D95613, 1),
    (9223372036854775807, 1001, 1e-6, 0x18941BE08D5FE831, 1),
    (9223372036854775807, 1099511627782, 0.25, 0x8A7413659074E923, 0),
    (9223372036854775807, 1, 0.9999, 0x8BA00A5C98D95613, 0),
    (9223372036854775808, 4, 0.9999, 0xDF3010E653FBA130, 0),
    (9223372036854775808, 123456789, 0.1, 0xE59D5431D21D7E5C, 1),
    (9223372036854775808, 0, 0.5, 0xEBA9B089647466C2, 0),
    (9223372036854775808, 2, 1e-6, 0xEBA9B089647466C2, 1),
    (9223372036854775815, 1001, 1e-6, 0x77723E6478D90776, 1),
    (9223372036854775815, 1099511627782, 0.25, 0xD2A79B26B00AFA62, 1),
    (9223372036854775815, 1, 0.9999, 0x9EA1D3624754EF3E, 0),
    (9223372036854775815, 3, 0.1, 0x9EA1D3624754EF3E, 1),
    (18446744073709551615, 123456789, 0.1, 0x6F9A643A3484BEC6, 1),
    (18446744073709551615, 0, 0.5, 0xD542C30584151160, 0),
    (18446744073709551615, 2, 1e-6, 0xD542C30584151160, 1),
    (18446744073709551615, 4, 0.25, 0x378ED17699F86172, 1),
    (18446744073709551600, 1099511627782, 0.25, 0xA4430717B9BBD866, 0),
    (18446744073709551600, 1, 0.9999, 0x256891ECEDB5343F, 0),
    (18446744073709551600, 3, 0.1, 0x256891ECEDB5343F, 1),
    (18446744073709551600, 1001, 0.5, 0x46E264BA91418ACE, 1),
]

# p -> (esp_dropout_thresh(p), esp_dropout_scale(p)); p = 1 is the clamp to 65535
THRESH_SCALE = {1e-6: (0, 1.0), 0.1: (6554, 1.11111867), 0.25: (16384, 1.33333337), 0.5: (32768, 2.0),
                0.9999: (65529, 9362.28613), 1.0: (65535, 65536.0)}


def test_hash_and_keep_known_answers():
    for seed, idx, p, h, k in KNOWN:
        assert int(R.hash_u64(seed, idx >> 2)) == h, (seed, idx)
        assert bool(R.keep(seed, idx, p)) == bool(k), (seed, idx, p)
    # vectorised: the same answers from one call per seed over an index array
    for seed in sorted({s for s, *_ in KNOWN}):
        rows = [(i, h) for s, i, _, h, _ in KNOWN if s == seed]
        idx = np.array([i for i, _ in rows], dtype=np.uint64)
        assert [int(v) for v in R.hash_u64(seed, idx >> np.uint64(2))] == [h for _, h in rows]


def test_lanes_of_a_group_share_one_hash():
    """idx 4g .. 4g+3 read the four 16-bit lanes of hash(seed, g), lowest lane first."""
    seed = 0xFFFFFFFFFFFFFFF0
    h = int(R.hash_u64(seed, 7))
    lanes = [(h >> (16 * t)) & 0xFFFF for t in range(4)]
    for p in (0.1, 0.5, 0.9):
        t = R.thresh(p)
        assert list(R.keep(seed, np.arange(28, 32), p)) == [lane >= t for lane in lanes]


@pytest.mark.parametrize("p", sorted(THRESH_SCALE))
def test_thresh_and_scale(p):
    t, s = THRESH_SCALE[p]
    assert R.thresh(p) == t
    assert np.float32(R.scale(p)) == np.float32(s)
    assert R.scale(p) == float(np.float32(65536.0 / (65536.0 - t)))
    if t == 0:  # nothing is dropped and nothing rescaled
        assert R.keep(3, np.arange(4096), p).all() and R.scale(p) == 1.0
    assert R.thresh(0.0) == 0 and R.scale(0.0) == 1.0


def test_device_seed_wraps_modulo_2_64():
    assert R.combine_seed(5, 2 ** 64 - 3) == 2
    assert R.combine_seed(2 ** 63, 2 ** 63) == 0
    assert R.combine_seed(7, -1) == 6            # an int64 device tensor holding -1 is 2^64 - 1
    idx = np.arange(1000)
    assert (R.keep(R.combine_seed(5, 2 ** 64 - 3), idx, 0.3) == R.keep(2, idx, 0.3)).all()


def test_keep_rate_and_no_float_promotion():
    idx = np.arange(1 << 16, dtype=np.int64) + (1 << 40)
    k = R.keep(2 ** 64 - 1, idx, 0.1)
    assert k.dtype == np.bool_ and abs(k.mean() - 0.9) < 0.005
    m = R.keep_mask(11, torch.arange(64).view(8, 8), 0.5)
    assert m.dtype == torch.bool and m.shape == (8, 8)
    assert torch.equal(m.reshape(-1), torch.from_numpy(R.keep(11, np.arange(64), 0.5)))
