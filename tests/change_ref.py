"""The edge changes of docs/SPEC.md §18 in numpy float64: the reference the GPU tests of alz_edge_changes*,
alz_edge_changes_top* and alz_debug_edge_changes_rows compare against, bit for bit.

The union of a source's rows and a baseline's rows is matched by packed key (§3), in ascending key order, and
filtered by a presence mask. Each side's value is the §17 value of one metric (metric_ref.values); for COUNT and ERR5XX
it is divided by the side's windows (one rounding). A side where the row is absent gives 0. The change is DELTA
value - base, DROP base - value, or RATIO value / base (base = 0: +inf when value > 0, else 1.0), each one rounding.
The top changes rank as metric_ref.top ranks values, over the filtered list's changes."""
import numpy as np

import metric_ref as mr
from alaz_b200 import abi

ABSENT = abi.ABSENT


def row_keys(rows):
    """§3 packed keys of EDGE_OUT rows (alz_device.cuh row_key_of)."""
    ft = rows["from_type"].astype(np.uint64)
    tt = rows["to_type"].astype(np.uint64)
    f = rows["from"].astype(np.uint64)
    t = rows["to"].astype(np.uint64)
    m29 = np.uint64(0x1FFFFFFF)
    pod = (tt << np.uint64(61)) | ((f & m29) << np.uint64(32)) | t
    rev = np.uint64(1 << 63) | (ft << np.uint64(61)) | ((t & m29) << np.uint64(32)) | f
    return np.where(ft == abi.NODE_POD, pod, rev).astype(np.uint64)


def side_values(rows, spec, windows):
    """The §18 value of every row of one side."""
    v = mr.values(rows, spec)
    kind = spec[0] if isinstance(spec, tuple) else spec
    if kind in (abi.METRIC_COUNT, abi.METRIC_ERR5XX):
        v = v / np.float64(windows)
    return v


def change_of(mode, cur, base):
    cur, base = np.asarray(cur, dtype=np.float64), np.asarray(base, dtype=np.float64)
    if mode == abi.CHANGE_DELTA:
        return cur - base
    if mode == abi.CHANGE_DROP:
        return base - cur
    if mode == abi.CHANGE_RATIO:
        with np.errstate(divide="ignore", invalid="ignore"):
            q = cur / np.where(base > 0, base, 1.0)
        return np.where(base > 0, q, np.where(cur > 0, np.inf, 1.0))
    raise ValueError(mode)


def changes(src, base, spec, mode, presence, src_windows=1, base_windows=1):
    """(EDGE_CHANGE records of the filtered union in ascending key order, info dict with above = 0). src and base are
    EDGE_OUT arrays, each strictly ascending by packed key."""
    ka, kb = row_keys(src), row_keys(base)
    assert np.all(ka[1:] > ka[:-1]) and np.all(kb[1:] > kb[:-1]), "each side must be strictly ascending"
    va, vb = side_values(src, spec, src_windows), side_values(base, spec, base_windows)
    keys = np.union1d(ka, kb)
    ia = np.searchsorted(ka, keys)
    ib = np.searchsorted(kb, keys)
    in_a = (ia < len(ka)) & (ka[np.minimum(ia, max(len(ka) - 1, 0))] == keys) if len(ka) else np.zeros(len(keys), bool)
    in_b = (ib < len(kb)) & (kb[np.minimum(ib, max(len(kb) - 1, 0))] == keys) if len(kb) else np.zeros(len(keys), bool)
    pres = np.where(in_a & in_b, abi.PRESENT_BOTH, np.where(in_a, abi.PRESENT_NEW, abi.PRESENT_GONE)).astype(np.uint8)
    keep = (pres & np.uint8(presence)) != 0
    out = np.zeros(int(keep.sum()), dtype=abi.EDGE_CHANGE)
    ia, ib, in_a, in_b, pres = ia[keep], ib[keep], in_a[keep], in_b[keep], pres[keep]
    out["presence"] = pres
    out["index"] = np.where(in_a, ia, ABSENT)
    out["base_index"] = np.where(in_b, ib, ABSENT)
    ra = src[np.minimum(ia, max(len(src) - 1, 0))] if len(src) else None
    rb = base[np.minimum(ib, max(len(base) - 1, 0))] if len(base) else None
    for f in ("from_type", "to_type", "from", "to"):
        a = ra[f] if ra is not None else np.zeros(len(out), out.dtype[f])
        b = rb[f] if rb is not None else np.zeros(len(out), out.dtype[f])
        out[f] = np.where(in_a, a, b)
    out["value"] = np.where(in_a, va[np.minimum(ia, max(len(va) - 1, 0))] if len(va) else 0.0, 0.0)
    out["base_value"] = np.where(in_b, vb[np.minimum(ib, max(len(vb) - 1, 0))] if len(vb) else 0.0, 0.0)
    out["change"] = change_of(mode, out["value"], out["base_value"])
    both = int(np.isin(ka, kb).sum())
    info = dict(source_rows=len(src), base_rows=len(base), both=both, added=len(src) - both, gone=len(base) - both,
                listed=len(out), above=0, source_windows=int(src_windows), base_windows=int(base_windows))
    return out, info


def top(src, base, spec, mode, presence, k, min_change, src_windows=1, base_windows=1):
    """(the first min(k, above) records by change in rank order, info dict with above set)."""
    lst, info = changes(src, base, spec, mode, presence, src_windows, base_windows)
    idx, above = mr.top(lst["change"], k, min_change)
    info = dict(info, above=above)
    return lst[idx], info
