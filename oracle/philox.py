"""Oracle: the library's counter-based generator, restated in NumPy.

Test infrastructure only (see oracle/__init__.py).

Restates ``dmosopt_b200/csrc/common.cuh`` (``Philox``, ``u01_53``) and ``csrc/variation.cu`` (``u01_open``, ``ctr_hi``)
word for word, so that every draw a kernel makes can be recomputed on the host from (seed, stream_id, purpose, index):
  * key words   k0 = low 32 bits of the seed, k1 = high 32 bits;
  * counter     c0 / c1 = low / high word of ``ctr_lo``, c2 / c3 = low / high word of ``ctr_hi``;
  * ten rounds of Philox4x32 (Salmon, Moraes, Dror, Shaw 2011) with multipliers 0xD2511F53 / 0xCD9E8D57 and Weyl key
    increments 0x9E3779B9 / 0xBB67AE85.
The kernels key the high counter word by ``(stream_id << 8) | purpose`` and the low one by the element index.
"""

import numpy as np

M0 = np.uint64(0xD2511F53)
M1 = np.uint64(0xCD9E8D57)
W0 = np.uint64(0x9E3779B9)
W1 = np.uint64(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)
_32 = np.uint64(32)

# the purposes of csrc/variation.cu (enum Purpose) and of the grouped mutation (csrc/moea_ext.cu, csrc/smpso.cu)
P_TOURNAMENT, P_DECIDE, P_PAIR, P_SINGLE, P_GENES = 1, 2, 3, 4, 5
P_MUT_PARENT, P_MUT_GENES = 11, 12


def _u64(a):
    return np.asarray(a, dtype=np.uint64)


def philox4x32_10(seed, ctr_lo, ctr_hi):
    """The four output words (uint32 arrays, broadcast over ``ctr_lo`` / ``ctr_hi``) of ``Philox(seed)(ctr_lo, ctr_hi)``."""
    seed = int(seed) & (2**64 - 1)
    lo, hi = np.broadcast_arrays(_u64(ctr_lo), _u64(ctr_hi))
    c0, c1 = lo & _LO, lo >> _32
    c2, c3 = hi & _LO, hi >> _32
    a, b = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    for _ in range(10):
        p0 = M0 * c0  # 32 x 32 -> 64 bits: exact in uint64
        p1 = M1 * c2
        c0, c1, c2, c3 = (p1 >> _32) ^ c1 ^ a, p1 & _LO, (p0 >> _32) ^ c3 ^ b, p0 & _LO
        a = (a + W0) & _LO
        b = (b + W1) & _LO
    return tuple(w.astype(np.uint32) for w in (c0, c1, c2, c3))


def ctr_hi(stream_id, purpose):
    """The high counter word of a draw: ``(stream_id << 8) | purpose`` (64-bit wrap-around, as on the device)."""
    return np.uint64(((int(stream_id) << 8) | int(purpose)) & (2**64 - 1))


def _mantissa53(hi, lo):
    return ((_u64(hi) >> np.uint64(5)) << np.uint64(26)) | (_u64(lo) >> np.uint64(6))


def u01_53(hi, lo):
    """53-bit uniform in [0, 1) from two words (common.cuh; the construction of numpy's Generator.random)."""
    return _mantissa53(hi, lo).astype(np.float64) * (1.0 / 9007199254740992.0)


def u01_open(hi, lo):
    """Uniform in the open interval (0, 1): the 53-bit grid shifted by half a step (variation.cu)."""
    return (_mantissa53(hi, lo).astype(np.float64) + 0.5) * (1.0 / 9007199254740992.0)


def draws(seed, stream_id, purpose, index):
    """``Philox(seed)(index, ctr_hi(stream_id, purpose))`` for an array of indices."""
    return philox4x32_10(seed, index, ctr_hi(stream_id, purpose))
