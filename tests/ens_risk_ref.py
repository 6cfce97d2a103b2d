"""The worst-m score of a planner ensemble (DESIGN.md §5m) restated in numpy: the specification k_ens_worst is held to."""
import numpy as np

from tests.ens_ref import ordered_mean

f32 = np.float32
NAN = np.uint32(0x7FFFFFFF).view(f32)   # the one NaN the score writes


def worst_m(r: np.ndarray, m: int) -> np.ndarray:
    """r [..., K] member returns -> [...] sample returns.  m = 0: the ordered mean.  1 <= m <= K: NaN (0x7fffffff) if any return of
    the row is NaN; otherwise the K returns sorted ascending with ties broken by member index (so -0 and +0 keep the members'
    order), s = r_(0), s = fl(s + r_(j)) for j = 1 .. m - 1, and fl(s / m), a NaN result (-inf + inf) written as 0x7fffffff too"""
    r = np.asarray(r, dtype=f32)
    K = r.shape[-1]
    if m == 0:
        return ordered_mean(r.reshape(-1, K)).reshape(r.shape[:-1])
    if not 1 <= m <= K:
        raise ValueError(f"m must be in 0 .. K = {K} (got {m})")
    flat = r.reshape(-1, K)
    srt = np.take_along_axis(flat, np.argsort(flat, axis=1, kind="stable"), axis=1)   # stable: equal values keep member order
    s = srt[:, 0].copy()
    with np.errstate(over="ignore", invalid="ignore"):
        for j in range(1, m):
            s = (s + srt[:, j]).astype(f32)
        s = (s / f32(m)).astype(f32)
    s[np.isnan(s) | np.isnan(flat).any(axis=1)] = NAN
    return s.reshape(r.shape[:-1])
