"""The top anomalous rows of docs/SPEC.md §16 in numpy: the reference the GPU tests of alz_gnn_top* and
alz_debug_top_scores compare against, bit for bit.

Each float32 score maps to a 32-bit key: bits u -> u ^ 0x80000000 when the sign bit is clear, ~u when it is set (IEEE
total order: -0 < +0, NaNs at the ends). Rows rank by key descending, then by index ascending; a row is eligible when
key(score) >= key(min_score); the result is the first min(k, above) eligible rows in rank order."""
import numpy as np


def order_key(scores):
    """uint32 keys of float32 scores (an array or a scalar)."""
    u = np.asarray(scores, dtype=np.float32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u ^ np.uint32(0x80000000)).astype(np.uint32)


def top_lexsort(scores, k, min_score):
    """The definition, spelled out: lexsort((index, -key)), filter, cut at k. (indices uint32, above)."""
    key = order_key(scores).astype(np.int64)
    idx = np.arange(len(key))
    order = np.lexsort((idx, -key))
    kmin = int(order_key(np.float32(min_score)))
    elig = order[key[order] >= kmin]
    return elig[:k].astype(np.uint32), len(elig)


def top(scores, k, min_score):
    """The same result by a partial sort of (~key << 32 | index), for arrays of up to 2^30 scores."""
    key = order_key(scores)
    n = len(key)
    above = int(np.count_nonzero(key >= order_key(np.float32(min_score))))
    m = min(int(k), above)
    if m == 0:
        return np.zeros(0, np.uint32), above
    comp = ((~key).astype(np.uint64) << np.uint64(32)) | np.arange(n, dtype=np.uint64)
    sel = np.argpartition(comp, m - 1)[:m] if m < n else np.arange(n)
    sel = sel[np.argsort(comp[sel], kind="stable")]
    return sel.astype(np.uint32), above
