"""numpy float64 restatement of docs/SPEC.md §6 (GNN anomaly pass). TEST INFRASTRUCTURE ONLY:
the oracle for alz_gnn_score. Shares no code with alaz_b200/csrc/alz_gnn.cu."""
import numpy as np
from scipy import sparse

M64 = (1 << 64) - 1
SEED = 0xA1A26E6E
D = 64


def splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def unit(idx):
    return (splitmix64(SEED + idx) >> 11) * (1.0 / 9007199254740992.0) * 2.0 - 1.0


def weights():
    sw, sa = 1.0 / np.sqrt(128.0), 1.0 / np.sqrt(132.0)
    idx = 0
    W, b = [], []
    for _ in range(2):
        w = np.zeros((128, D), dtype=np.float32)
        for k in range(128):
            for j in range(D):
                w[k, j] = np.float32(unit(idx) * sw)
                idx += 1
        bb = np.zeros(D, dtype=np.float32)
        for j in range(D):
            bb[j] = np.float32(unit(idx) * 0.01)
            idx += 1
        W.append(w.astype(np.float64))
        b.append(bb.astype(np.float64))
    a = np.zeros(132, dtype=np.float32)
    for k in range(132):
        a[k] = np.float32(unit(idx) * sa)
        idx += 1
    return W, b, a.astype(np.float64), 0.0


def bucket_lo(b):
    if b == 0:
        return 0.0
    base = float(1 << (8 + b // 2))
    return base * 1.5 if b & 1 else base


def bucket_hi(b):
    return float(1 << 40) if b == 63 else bucket_lo(b + 1)


def quantile(hist, q):
    total = int(np.sum(hist.astype(np.uint64)))
    if total == 0:
        return 0.0
    target = q * float(total)
    cum = 0.0
    for b in range(64):
        c = float(hist[b])
        if c > 0.0 and cum + c >= target:
            f = max((target - cum) / c, 0.0)
            return bucket_lo(b) + f * (bucket_hi(b) - bucket_lo(b))
        cum += c
    return bucket_hi(63)


_LO = np.array([bucket_lo(b) for b in range(64)])
_HI = np.array([bucket_hi(b) for b in range(64)])


def quantiles_vec(hist, q):
    """quantile() for every row of hist at once (same arithmetic, float64)."""
    h = hist.astype(np.float64)
    total = h.sum(axis=1)
    target = q * total
    cum = np.cumsum(h, axis=1)
    ok = (h > 0.0) & (cum >= target[:, None])
    b = np.argmax(ok, axis=1)
    any_ok = ok.any(axis=1)
    rows = np.arange(len(h))
    before = cum[rows, b] - h[rows, b]
    c = np.where(h[rows, b] > 0.0, h[rows, b], 1.0)
    f = np.maximum((target - before) / c, 0.0)
    val = _LO[b] + f * (_HI[b] - _LO[b])
    val = np.where(any_ok, val, _HI[63])
    return np.where(total > 0.0, val, 0.0)


def _graph(edges):
    """Node keys, edge ends (u, v) and the float32-stored features h0 (SPEC §6). The per-node sums of count,
    5xx and latency are u64 and wrap mod 2^64 like the edge accumulators (SPEC §3); they become float64 only
    for the features."""
    fk = (edges["from_type"].astype(np.uint64) << np.uint64(32)) | edges["from"].astype(np.uint64)
    tk = (edges["to_type"].astype(np.uint64) << np.uint64(32)) | edges["to"].astype(np.uint64)
    nodes = np.unique(np.concatenate([fk, tk]))
    n_v = len(nodes)
    u = np.searchsorted(nodes, fk)
    v = np.searchsorted(nodes, tk)
    st = np.zeros((n_v, 8), dtype=np.uint64)
    for k, f in enumerate(("count", "err5xx", "lat_sum_ns")):
        x = edges[f].astype(np.uint64)
        np.add.at(st[:, 2 * k], u, x)        # uint64 adds: mod 2^64
        np.add.at(st[:, 2 * k + 1], v, x)
    np.add.at(st[:, 6], u, np.uint64(1)); np.add.at(st[:, 7], v, np.uint64(1))
    st = st.astype(np.float64)

    def ratio(a, b):
        return np.divide(a, b, out=np.zeros_like(a), where=b > 0)
    kind = (nodes >> np.uint64(32)).astype(np.int64)
    h = np.zeros((n_v, D), dtype=np.float64)
    h[:, 0] = np.log1p(st[:, 0]); h[:, 1] = np.log1p(st[:, 1])
    h[:, 2] = ratio(st[:, 2], st[:, 0]); h[:, 3] = ratio(st[:, 3], st[:, 1])
    h[:, 4] = np.log1p(ratio(st[:, 4], st[:, 0])); h[:, 5] = np.log1p(ratio(st[:, 5], st[:, 1]))
    h[:, 6] = np.log1p(st[:, 6]); h[:, 7] = np.log1p(st[:, 7])
    h[:, 8] = kind == 0; h[:, 9] = kind == 1; h[:, 10] = kind >= 2; h[:, 11] = 1.0   # outbound, by address or by Host header
    h = h.astype(np.float32).astype(np.float64)   # features are stored as float32
    return nodes, u, v, st[:, 7], h


def _layers(h, u, v, indeg, W, b):
    """Two GraphSAGE-mean layers; the neighbour means are float64 sums (SPEC §6)."""
    n_v = len(h)
    # A[v, u] = 1 per edge u -> v: the neighbour sums as one sparse product, float64
    A = sparse.csr_matrix((np.ones(len(u)), (v, u)), shape=(n_v, n_v))
    for l in range(2):
        m = np.asarray(A @ h)
        m = np.divide(m, indeg[:, None], out=np.zeros_like(m), where=indeg[:, None] > 0)
        z = np.concatenate([h, m], axis=1)
        h = np.maximum(z @ W[l] + b[l], 0.0)
    return h


def run(edges, with_scale=False):
    """edges: alz_edge_out array (any order). Returns (node_keys, h2, scores) with scores in the input order.
    with_scale: also the magnitude pass, the same two layers on |h0|, |W| and |b|: for every element of h2, the sum
    of the absolute values of every term that went into it (the scale an elementwise error bound refers to)."""
    n_e = len(edges)
    nodes, u, v, indeg, h0 = _graph(edges)
    W, b, a, c = weights()
    h = _layers(h0, u, v, indeg, W, b)
    cnt = edges["count"].astype(np.float64)
    err = edges["err5xx"].astype(np.float64)
    e_feat = np.zeros((n_e, 4), dtype=np.float64)
    e_feat[:, 0] = np.log1p(cnt)
    e_feat[:, 1] = np.divide(err, cnt, out=np.zeros_like(err), where=cnt > 0)
    e_feat[:, 2] = np.log1p(quantiles_vec(edges["hist"], 0.5))
    e_feat[:, 3] = np.log1p(quantiles_vec(edges["hist"], 0.99))
    zz = np.concatenate([h[u], h[v], e_feat], axis=1) @ a + c
    scores = 1.0 / (1.0 + np.exp(-zz))
    if not with_scale:
        return nodes, h, scores
    scale = _layers(np.abs(h0), u, v, indeg, [np.abs(w) for w in W], [np.abs(x) for x in b])
    return nodes, h, scores, scale
