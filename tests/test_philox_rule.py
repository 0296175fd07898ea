"""tests/philox_rule.py on the CPU: the vectorised rule against a scalar transcription of csrc/common.cuh, its keep
rate, the independence of its sites, seeds and rows, and the 64-bit carry of seed + counter."""
import numpy as np
import pytest

import philox_rule as R


def _philox_scalar(c0, c1, c2, c3, k0, k1):
    """common.cuh philox4, line by line, on Python ints"""
    M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
    m = 0xFFFFFFFF
    for _ in range(7):
        hi0, lo0 = (M0 * c0) >> 32, (M0 * c0) & m
        hi1, lo1 = (M1 * c2) >> 32, (M1 * c2) & m
        n0, n2 = hi1 ^ c1 ^ k0, hi0 ^ c3 ^ k1
        c0, c1, c2, c3 = n0, lo1, n2, lo0
        k0, k1 = (k0 + W0) & m, (k1 + W1) & m
    return c0, c1, c2, c3


def _keep8_scalar(seed, stream, idx8, p):
    """common.cuh dropout_keep8 on Python ints (seed already includes the counter, mod 2^64)"""
    r = _philox_scalar(idx8 & 0xFFFFFFFF, idx8 >> 32, stream, 0, seed & 0xFFFFFFFF, seed >> 32)
    thr = int(np.float32(p) * np.float32(65536.0))
    m = 0
    for j in range(4):
        m |= int((r[j] & 0xFFFF) >= thr) << (2 * j)
        m |= int((r[j] >> 16) >= thr) << (2 * j + 1)
    return m


SEEDS = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 62 - 1, 2 ** 64 - 1, 0x0123456789ABCDEF]


def test_philox_matches_the_scalar_transcription():
    rng = np.random.default_rng(0)
    c = rng.integers(0, 2 ** 32, (4, 64), dtype=np.uint64)
    k = rng.integers(0, 2 ** 32, (2, 64), dtype=np.uint64)
    c[:, 0] = 0
    c[:, 1] = 2 ** 32 - 1
    k[:, 2] = 2 ** 32 - 1
    for i in range(64):
        got = R.philox4x32_7(c[0, i], c[1, i], c[2, i], c[3, i], k[0, i], k[1, i])
        ref = _philox_scalar(*(int(v) for v in c[:, i]), int(k[0, i]), int(k[1, i]))
        assert tuple(int(g) for g in got) == ref, i
    # vectorised call over the whole batch at once
    got = R.philox4x32_7(c[0], c[1], c[2], c[3], k[0], k[1])
    for i in range(64):
        assert tuple(int(g[i]) for g in got) == _philox_scalar(*(int(v) for v in c[:, i]), int(k[0, i]), int(k[1, i]))


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("p", [0.1, 0.2, 0.3])
def test_keep_mask_matches_the_scalar_rule(seed, p):
    rows = np.array([0, 1, 7, 41599, 2 ** 27 + 3])               # row * 32 + lane crosses 2^32: the high counter word
    stream, ctr = 77, 5
    m = R.keep_mask(seed, ctr, stream, rows, p)
    key = (seed + ctr) % 2 ** 64
    for a, r in enumerate(rows):
        for lane in range(32):
            k8 = _keep8_scalar(key, stream, int(r) * 32 + lane, p)
            for i in range(8):
                assert bool(m[a, 8 * lane + i]) == bool((k8 >> i) & 1), (r, lane, i)


def test_threshold_is_computed_in_fp32():
    assert R.threshold(0.1) == 6553 and R.threshold(0.2) == 13107 and R.threshold(0.3) == 19660
    assert R.keep_scale(0.1) == 1.0 / (1.0 - float(np.float32(0.1)))


@pytest.mark.parametrize("p", [0.1, 0.2, 0.3])
def test_keep_rate(p):
    n = 4096 * 256
    m = R.keep_mask(987654321, 0, 3, 4096, p)
    q = 1.0 - R.threshold(p) / 65536.0
    sigma = np.sqrt(q * (1 - q) / n)
    assert abs(m.mean() - q) <= 4 * sigma, (m.mean(), q, sigma)


def _agreement_ok(a, b, p):
    """two independent keep masks agree on a fraction q^2 + (1-q)^2 of the elements"""
    q = 1.0 - R.threshold(p) / 65536.0
    e = q * q + (1 - q) * (1 - q)
    n = a.size
    agree = (a == b).mean()
    return abs(agree - e) <= 4 * np.sqrt(e * (1 - e) / n), (agree, e)


def test_sites_seeds_and_rows_are_independent():
    p = 0.2
    base = R.keep_mask(12345, 0, R.encoder_sid(0, 0, "gcn_ln"), 2048, p)
    others = {
        "next site": R.keep_mask(12345, 0, R.encoder_sid(0, 0, "comb_ln"), 2048, p),
        "next layer": R.keep_mask(12345, 0, R.encoder_sid(0, 1, "gcn_ln"), 2048, p),
        "decoder site": R.keep_mask(12345, 0, R.decoder_sid(0, 0, "ffn"), 2048, p),
        "next seed": R.keep_mask(12346, 0, R.encoder_sid(0, 0, "gcn_ln"), 2048, p),
        "next counter": R.keep_mask(12345, 1, R.encoder_sid(0, 0, "gcn_ln"), 2048, p),
        "seed high word": R.keep_mask(12345 + 2 ** 32, 0, R.encoder_sid(0, 0, "gcn_ln"), 2048, p),
        "shifted rows": R.keep_mask(12345, 0, R.encoder_sid(0, 0, "gcn_ln"), np.arange(1, 2049), p),
    }
    for what, m in others.items():
        ok, info = _agreement_ok(base, m, p)
        assert ok, (what, info)
    # the 8 elements of one lane come from one draw: neighbouring bits must be independent too
    ok, info = _agreement_ok(base[:, 0::2], base[:, 1::2], p)
    assert ok, ("adjacent elements", info)


def test_seed_counter_carries_into_the_high_word():
    a = R.keep_mask(2 ** 32 - 1, 1, 5, 64, 0.1)
    b = R.keep_mask(2 ** 32, 0, 5, 64, 0.1)
    assert np.array_equal(a, b)
    assert np.array_equal(R.keep_mask(2 ** 64 - 1, 1, 5, 64, 0.1), R.keep_mask(0, 0, 5, 64, 0.1))    # mod 2^64
    assert not np.array_equal(a, R.keep_mask(0, 0, 5, 64, 0.1))                                  # not dropped


def test_sample_uniform_matches_the_scalar_transcription():
    seed = 0xDEADBEEF12345678
    for first, b, n, pos in [(0, 0, 0, 0), (7, 2, 3, 5), (2 ** 31 - 4, 3, 31, 29)]:
        x = _philox_scalar(first + b, n, 0x53414D50, pos, seed & 0xFFFFFFFF, seed >> 32)[0]
        assert R.sample_uniform(seed, first, b, n, pos) == (x >> 8) * 2.0 ** -24
    u = R.sample_uniform(seed, 0, np.arange(4096), 0, 1)
    assert 0.0 <= u.min() and u.max() < 1.0 and abs(u.mean() - 0.5) < 4 * np.sqrt(1 / 12 / 4096)
