"""Host-side JAX-compatible PRNG key management (threefry2x32, legacy non-partitionable layout).

Mirrors what the reference gets from `jax.random.PRNGKey / split / uniform`
(upstream mbd/planners/mbd_planner.py:40,79,103,150; envs/humanoidrun.py:21-27).
Only key bookkeeping and the 47 reset-noise uniforms run here (once per solve); the bulk
`jax.random.normal` of `reverse_once` is generated on the GPU (csrc/mbd_kernels.cu).
Known-answer vectors from JAX's own test-suite are checked in tests/test_prng.py.
"""
from __future__ import annotations

import numpy as np

_ROT = ((13, 15, 26, 6), (17, 29, 16, 24))
_M32 = np.uint64(0xFFFFFFFF)


def _rotl(x, r):
    return ((x << np.uint32(r)) | (x >> np.uint32(32 - r))).astype(np.uint32)


def threefry2x32(key, c0, c1):
    """Vectorised threefry2x32: key uint32[2]; c0, c1 uint32 arrays -> (o0, o1)."""
    with np.errstate(over="ignore"):
        k0, k1 = np.uint32(key[0]), np.uint32(key[1])
        ks = [k0, k1, np.uint32(k0 ^ k1 ^ np.uint32(0x1BD11BDA))]
        x0 = (np.asarray(c0, dtype=np.uint32) + ks[0]).astype(np.uint32)
        x1 = (np.asarray(c1, dtype=np.uint32) + ks[1]).astype(np.uint32)
        for i in range(5):
            for r in _ROT[i % 2]:
                x0 = (x0 + x1).astype(np.uint32)
                x1 = _rotl(x1, r) ^ x0
            x0 = (x0 + ks[(i + 1) % 3]).astype(np.uint32)
            x1 = (x1 + ks[(i + 2) % 3] + np.uint32(i + 1)).astype(np.uint32)
    return x0, x1


_PARTITIONABLE = False


def set_layout(partitionable: bool):
    """Threefry counter layout of this module AND of the in-kernel samplers (process-wide).  False (default): the legacy layout,
    `jax_threefry_partitionable=False`, pinned by JAX's known-answer vectors.  True: the partitionable layout that JAX >= 0.5 uses
    by default **[jax-recalled], unpinned**: `random_bits` element i = xor of the two output words of block (hi, lo) = (0, i);
    `split(key, n)[i]` = the two output words of block (0, i).  Also settable with MBD_THREEFRY_PARTITIONABLE=1."""
    global _PARTITIONABLE
    _PARTITIONABLE = bool(partitionable)
    from . import _lib
    _lib.check(_lib.lib().mbd_set_prng_layout(1 if partitionable else 0), "mbd_set_prng_layout")


def random_bits(key, total: int) -> np.ndarray:
    """jax.random.bits(key, (total,), uint32): counters iota(total) split in halves (odd -> zero pad)."""
    if _PARTITIONABLE:
        o0, o1 = threefry2x32(key, np.zeros(total, dtype=np.uint32), np.arange(total, dtype=np.uint32))
        return (o0 ^ o1).astype(np.uint32)
    half = (total + 1) // 2
    cnt = np.arange(2 * half, dtype=np.uint32)
    if total % 2:
        cnt[-1] = 0
    o0, o1 = threefry2x32(key, cnt[:half], cnt[half:])
    return np.concatenate([o0, o1])[:total]


def PRNGKey(seed: int) -> np.ndarray:
    return np.array([(int(seed) >> 32) & 0xFFFFFFFF, int(seed) & 0xFFFFFFFF], dtype=np.uint32)


def split(key, num: int = 2) -> np.ndarray:
    if _PARTITIONABLE:
        o0, o1 = threefry2x32(key, np.zeros(num, dtype=np.uint32), np.arange(num, dtype=np.uint32))
        return np.stack([o0, o1], axis=1).astype(np.uint32)
    return random_bits(key, 2 * num).reshape(num, 2)


def uniform(key, shape, minval=0.0, maxval=1.0) -> np.ndarray:
    total = int(np.prod(shape)) if len(shape) else 1
    bits = random_bits(key, total)
    unit = ((bits >> np.uint32(9)) | np.uint32(0x3F800000)).view(np.float32) - np.float32(1.0)
    lo, hi = np.float32(minval), np.float32(maxval)
    return np.maximum(lo, unit * (hi - lo) + lo).astype(np.float32).reshape(shape)


def _threefry_int(k0: int, k1: int, c0: int, c1: int):
    """threefry2x32 on Python ints (one block) — the key chain of a solve is sequential, and for two-word inputs plain ints are
    ~10x faster than numpy scalars"""
    M = 0xFFFFFFFF
    ks = (k0, k1, k0 ^ k1 ^ 0x1BD11BDA)
    x0, x1 = (c0 + ks[0]) & M, (c1 + ks[1]) & M
    for i in range(5):
        for r in _ROT[i % 2]:
            x0 = (x0 + x1) & M
            x1 = (((x1 << r) | (x1 >> (32 - r))) & M) ^ x0
        x0 = (x0 + ks[(i + 1) % 3]) & M
        x1 = (x1 + ks[(i + 2) % 3] + i + 1) & M
    return x0, x1


def fold_in(key, data: int) -> np.ndarray:
    """jax.random.fold_in(key, data) **[jax-recalled]**: threefry2x32(key, (0, data))"""
    return np.array(_threefry_int(int(key[0]), int(key[1]), 0, int(data) & 0xFFFFFFFF), np.uint32)


def split2(key):
    """split(key, 2) for the planner's `rng, Y0s_rng = split(rng)` chain: returns (new_key, sub_key) as uint32[2] arrays"""
    k0, k1 = int(key[0]), int(key[1])
    if _PARTITIONABLE:
        return (np.array(_threefry_int(k0, k1, 0, 0), dtype=np.uint32), np.array(_threefry_int(k0, k1, 0, 1), dtype=np.uint32))
    a0, a1 = _threefry_int(k0, k1, 0, 2)     # counters iota(4) split in halves: blocks (0, 2) and (1, 3)
    b0, b1 = _threefry_int(k0, k1, 1, 3)
    return np.array([a0, b0], dtype=np.uint32), np.array([a1, b1], dtype=np.uint32)


import os as _os
if _os.environ.get("MBD_THREEFRY_PARTITIONABLE", "0") == "1":   # compatibility switch (ADVICE r1): match a JAX >= 0.5 install
    try:
        set_layout(True)
    except Exception:  # noqa: BLE001 - no library yet (first build): the flag is applied by the first explicit set_layout call
        _PARTITIONABLE = True
