"""CPU: the numpy restatement of the device RNG (oracle/philox.py) against plain-integer Philox arithmetic. The GPU
tests hold the kernels' draws against this restatement (tests/test_emulator_device_rng.py)."""
import numpy as np

import philox

MASK = 0xFFFFFFFF


def philox_int(ctr, key, rounds):
    """Philox4x32-R on Python integers, every operation reduced modulo 2^32 explicitly."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for _ in range(rounds):
        p0, p1 = philox.M0 * c0, philox.M1 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & MASK, p1 & MASK, ((p0 >> 32) ^ c3 ^ k1) & MASK, p0 & MASK
        k0, k1 = (k0 + philox.W0) & MASK, (k1 + philox.W1) & MASK
    return c0, c1, c2, c3


def test_known_answers_philox4x32_10():
    """Random123's published known-answer vectors for Philox4x32-10 (same round function, 10 rounds)."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((MASK, MASK, MASK, MASK), (MASK, MASK), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        got = philox.philox4x32(tuple(np.array([c], np.uint32) for c in ctr), key, rounds=10)
        assert tuple(int(g[0]) for g in got) == want


def test_matches_integer_arithmetic_with_wraparound():
    """Random counters and keys, including all-ones words (every product, xor and key bump wraps)."""
    rng = np.random.default_rng(1)
    ctr = [rng.integers(0, 2 ** 32, 2000, dtype=np.uint64).astype(np.uint32) for _ in range(4)]
    for c in ctr:
        c[:3] = MASK
    for key in ((0, 0), (MASK, MASK), (0x12345678, 0xFFFFFFF0)):
        got = philox.philox4x32(ctr, key)
        for i in range(0, 2000, 37):
            want = philox_int(tuple(int(c[i]) for c in ctr), key, philox.ROUNDS)
            assert tuple(int(g[i]) for g in got) == want


def test_consistent_across_round_counts():
    """R rounds == one more round, with the key bumped R - 1 times, applied to the output of R - 1 rounds."""
    rng = np.random.default_rng(2)
    ctr = [rng.integers(0, 2 ** 32, 500, dtype=np.uint64).astype(np.uint32) for _ in range(4)]
    key = (0xDEADBEEF, 0x0BADF00D)
    for r in range(1, 11):
        prev = philox.philox4x32(ctr, key, rounds=r - 1)
        bumped = ((key[0] + (r - 1) * philox.W0) & MASK, (key[1] + (r - 1) * philox.W1) & MASK)
        step = philox.philox4x32(prev, bumped, rounds=1)
        full = philox.philox4x32(ctr, key, rounds=r)
        assert all(np.array_equal(a, b) for a, b in zip(step, full)), r
    assert all(np.array_equal(a, b) for a, b in zip(philox.philox4x32(ctr, key, rounds=0), ctr))


def test_shot_uniform_is_prefix_then_truncated_low_bits():
    """float_rz((pref << 20) | (w >> 12)) * 2^-32: in [0, 1), never rounded up, top 12 bits = the prefix the kernels
    test against pref_lo; checked against exact integer truncation."""
    seed, n = (7 << 32) | 99, 4099
    for px_off in (0, 3):
        u = philox.shot_u01(seed, n, 5, px_off=px_off)
        assert u.dtype == np.float32 and u.min() >= 0 and u.max() < 1
        pref = philox.leak_fields(seed, n, 5, px_off=px_off)[3]
        assert np.array_equal(np.floor(u.astype(np.float64) * 4096).astype(np.uint32), pref)
        g = np.arange(n) + px_off
        w = philox.philox4x32((g >> 2, np.full(n, 5), np.full(n, 1), np.full(n, philox.TAG_SHOT)),
                              philox.seed_key(seed))
        for i in range(0, n, 41):
            v = (int(pref[i]) << 20) | (int(w[g[i] & 3][i]) >> 12)
            t = v if v < 2 ** 24 else (v >> (v.bit_length() - 24)) << (v.bit_length() - 24)
            assert float(u[i]) == t / 2.0 ** 32
    # a pixel offset that is not a multiple of 4 draws the matching slice of the offset-0 field
    full = philox.shot_u01(seed, n + 8, 5)
    assert np.array_equal(philox.shot_u01(seed, n, 5, px_off=3), full[3:3 + n])


def test_leak_prefix_layout_and_box_muller_inputs():
    """12-bit prefixes are the bits Box-Muller leaves over; the radius argument lies in (0, 1] (rounding of the
    fmaf may reach 1.0 exactly) and the normals have unit scale."""
    u, ang, sc, pref = philox.leak_fields(3, 1 << 16, 0)
    assert pref.max() < 4096 and u.min() > 0 and u.max() <= 1
    assert ang.min() >= 0 and ang.max() < 2 * np.pi
    x = philox.normals(u, ang, sc)
    assert abs(x.mean()) < 5 / 256 and abs(x.var() - 1) < 5 * np.sqrt(2) / 256
    # the prefix is spread evenly over its 4096 values (chi-square, 4095 dof, ~5 sigma)
    h = np.bincount(pref, minlength=4096)
    chi2 = ((h - 16.0) ** 2 / 16.0).sum()
    assert abs(chi2 - 4095) < 5 * np.sqrt(2 * 4095)
