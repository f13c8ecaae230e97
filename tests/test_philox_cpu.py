"""The NumPy restatement of the library's Philox4x32-10 (oracle/philox.py) against the generator's published answers.

The GPU tests replay the operator kernels' random draws through this restatement (tests/test_gpu_operators.py), and
check there that it reproduces the draws the kernels return, bit for bit."""

import numpy as np
import pytest

from oracle import philox


def words_to_u64(w0, w1):
    return np.uint64(w0) | (np.uint64(w1) << np.uint64(32))


# Random123's known-answer vectors for philox4x32-10: (counter words c0..c3, key words k0 k1) -> output words
KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,expect", KAT)
def test_known_answers(ctr, key, expect):
    seed = int(key[0]) | (int(key[1]) << 32)
    out = philox.philox4x32_10(seed, words_to_u64(ctr[0], ctr[1]), words_to_u64(ctr[2], ctr[3]))
    assert tuple(int(w) for w in out) == expect


def test_vectorised_equals_scalar():
    rng = np.random.default_rng(0)
    lo = rng.integers(0, 2**63, size=64, dtype=np.int64).astype(np.uint64) * np.uint64(2) + np.uint64(1)
    hi = rng.integers(0, 2**63, size=64, dtype=np.int64).astype(np.uint64)
    seed = 0xDEADBEEFCAFEF00D
    vec = np.stack(philox.philox4x32_10(seed, lo, hi))
    for i in range(64):
        one = np.stack(philox.philox4x32_10(seed, lo[i], hi[i]))
        assert np.array_equal(vec[:, i], one)
    # a broadcast high word is the same as a repeated one
    b = np.stack(philox.philox4x32_10(seed, lo, hi[0]))
    r = np.stack(philox.philox4x32_10(seed, lo, np.full(64, hi[0])))
    assert np.array_equal(b, r)


def test_uniform_conversions_at_their_ends():
    zero, ones = np.uint32(0), np.uint32(0xFFFFFFFF)
    assert philox.u01_53(zero, zero) == 0.0
    assert philox.u01_53(ones, ones) == 1.0 - 2.0**-53  # the largest double below 1
    assert philox.u01_53(zero, np.uint32(1 << 6)) == 2.0**-53  # the low word contributes its top 26 bits
    assert philox.u01_53(np.uint32(1 << 5), zero) == 2.0**-27
    assert philox.u01_open(zero, zero) == 2.0**-54
    # (2^53 - 1) + 0.5 is not a double: it rounds to even, 2^53, so the device's open uniform can reach 1.0 exactly
    top = philox.u01_open(ones, ones)
    assert top == 1.0
    # bits dropped by the conversion do not matter
    assert philox.u01_53(np.uint32(0x1F), np.uint32(0x3F)) == 0.0


def test_counter_words():
    assert philox.ctr_hi(0, philox.P_GENES) == np.uint64(5)
    assert philox.ctr_hi(3, philox.P_MUT_PARENT) == np.uint64((3 << 8) | 11)
    assert philox.ctr_hi(2**56 + 7, 1) == np.uint64((7 << 8) | 1)  # the shift wraps at 64 bits, as on the device
    # the high word feeds counter words c2 / c3: a change of stream changes every output word
    a = np.stack(philox.draws(9, 1, philox.P_DECIDE, np.arange(8)))
    b = np.stack(philox.draws(9, 2, philox.P_DECIDE, np.arange(8)))
    assert np.all(a != b)
