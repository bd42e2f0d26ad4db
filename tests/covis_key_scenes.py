"""Order-key maps for the covisibility graph and its readers (orbfe_covis_*), shared by tests/test_oracle_covis_keys.py and
tests/test_gpu_covis_keys.py.

Every orbfe_covis_* entry orders keyframes by the caller's 64-bit key, (uintptr_t)pKF in an integration.  The scenes name
keyframes by creation index k; a key map gives each k its key.  `keys(name, n)` is the uint64 array of the first n keys,
`rank(keys)` each keyframe's place in key order: the order in which the reference's own driver lays the KeyFrames out
(oracle.covis.RefCovis.set_kf_order), so that the reference decides the same order.

The maps and the wrong implementations each separates from the right one:
  small        k.  The control: the keys every other test uses.
  wrap32       pointer-like: a stride of 0x2B0 bytes from 0x55d3_xxxx_xxxx, the low word wrapping past 2^32 at k = n // 2.
               Monotone.  Separates comparing only the low words (the keys past the wrap would sort first).
  high_only    (k + 1) << 32 | 0x12345678: every low word equal.  Separates comparing only the low words (every key ties).
               Swapped halves keep this map's order, so it does not separate them.
  top          monotone from near 0 to exactly 2^64 - 1, straddling 2^63; the last keyframe holds 2^64 - 1.  Separates signed
               comparisons (the keys at or past 2^63 would sort first) and padding that ties with the maximal key.
  interleaved  high word 7 - k % 8, low word 0xFFFFFFFF - k.  Key order is neither creation order nor slot order: separates
               anything that orders by creation index or by slot where it should order by key, and swapped halves.
  random       seeded distinct values, 0 and 2^64 - 1 among them.  All of the above at once, at no particular place."""
import numpy as np

NAMES = ("small", "wrap32", "high_only", "top", "interleaved", "random")
MONOTONE = ("small", "wrap32", "high_only", "top")
MAX = (1 << 64) - 1
STRIDE = 0x2B0


def _small(n):
    return [k for k in range(n)]


def _wrap32(n):
    base = (0x55d3 << 32) + (1 << 32) - STRIDE * (n // 2)
    return [base + STRIDE * k for k in range(n)]


def _high_only(n):
    return [(k + 1) << 32 | 0x12345678 for k in range(n)]


def _top(n):
    if n == 1:
        return [MAX]
    step = MAX // (n - 1)
    return [MAX - (n - 1 - k) * step for k in range(n)]


def _interleaved(n):
    return [(7 - k % 8) << 32 | (0xFFFFFFFF - k) for k in range(n)]


def _random(n, seed=20261017):
    rng = np.random.default_rng(seed + n)
    out, seen = [], set()
    while len(out) < n:
        v = int(rng.integers(0, 1 << 63)) << 1 | int(rng.integers(0, 2))
        if v not in seen and v not in (0, MAX):
            seen.add(v)
            out.append(v)
    at = rng.permutation(n)
    out[int(at[0])] = MAX
    if n > 1:
        out[int(at[1])] = 0
    return out


_MAPS = dict(small=_small, wrap32=_wrap32, high_only=_high_only, top=_top, interleaved=_interleaved, random=_random)


def keys(name, n):
    """the keys of keyframes 0 .. n-1 under map `name` (uint64)"""
    v = _MAPS[name](int(n))
    assert len(set(v)) == len(v) and all(0 <= x <= MAX for x in v)
    return np.array(v, np.uint64)


def rank(key):
    """each keyframe's place in key order (int32): the reference's KeyFrame layout for these keys"""
    return np.argsort(np.argsort(np.asarray(key, np.uint64), kind="stable"), kind="stable").astype(np.int32)


def key_list(key, n):
    """keys of keyframes 0 .. n-1: the creation index when `key` is None (the scenes' own keys), else key[:n]"""
    return np.arange(n, dtype=np.uint64) if key is None else np.asarray(key, np.uint64)[:n]


def key_of(key, k):
    """the key of keyframe k as a Python int"""
    return int(k) if key is None else int(key[k])
