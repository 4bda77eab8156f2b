"""GPU: GNN anomaly pass (docs/SPEC.md §6) against the numpy float64 restatement (tests/gnn_ref.py).

Scores: 1e-5 relative + 1e-6 absolute, as SPEC §6 states. Layer-2 embeddings: elementwise against the scale of
each element (below). Every test runs on both layer paths: the wgmma layer (sage_layer_tc_kernel) and the FP32
FFMA layer that ALZ_GNN_SIMT=1 selects (sage_layer_kernel). Graphs are built edge by edge (tests/gnn_graphs.py)
so that node counts, in-degrees and histograms land where the kernels' tiles, rings and scans have edges."""
import ctypes as C

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import gnn_graphs as gg
import gnn_ref
import oracle_lib as ol
from alaz_b200 import abi, capi

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-5, 1e-6

# h2 error bound: |h2 - h2_ref| <= GAMMA * scale elementwise, where scale is gnn_ref's magnitude pass (the same
# network on |h0|, |W|, |b|: the sum of the absolute values of every term behind an element). Per layer, relative
# to that scale, with u = 2^-24 (fp32) and t = 2^-11 (the relative rounding of the tf32 split):
#   3xTF32 products: x = hi + lo with lo exact, then lo rounded to tf32 (error <= t*|lo| <= t^2*|x|); hi*hi + hi*lo
#     + lo*hi leaves out lo*lo and the two rounded lo's: <= 3 t^2 = 2^-20.4 of each product, so of the scale;
#   fp32 accumulation of 3 x 128 products and the bias: roundings of random sign, each <= u * |partial sum| <=
#     u * scale: ~sqrt(384 / 3) * u = 2^-20.5 of the scale (the worst case, 384 u, is never approached and would
#     hide the faults below);
#   fp32 storage of the neighbour mean (summed in float64, rounded once) and of h1: u each.
# Layer 1's error reaches layer 2 through |W2|, which is how the scale is built, so the layers add: about
# 2 * (2^-20.4 + 2^-20.5 + 2^-23) = 2^-18.4. GAMMA = 2^-18. Observed on an H100 (400 W) over every graph below:
# at most 2.6e-7 = 2^-21.9 of the scale on the wgmma path and 8.3e-8 on the FFMA path. Dropping one tf32 cross
# product (hi*lo or lo*hi) costs t * |lo / x| ~ 2^-13 of a product and was observed at 1.7e-5 to 1.4e-4 of the
# scale (>= 4 GAMMA) on every graph here; an fp32 neighbour sum over a hub of 10^5 identical rows at 6.5e-5, of
# 10^6 rows at 1e-3.
GAMMA = 2.0 ** -18


def use_path(monkeypatch, path):
    """Select the layer path for the handles a test creates: a handle reads ALZ_GNN_SIMT at its first GNN call."""
    if path == "simt":
        monkeypatch.setenv("ALZ_GNN_SIMT", "1")
    else:
        monkeypatch.delenv("ALZ_GNN_SIMT", raising=False)
    return path


@pytest.fixture(params=["tc", "simt"])
def path(request, monkeypatch):
    return use_path(monkeypatch, request.param)


def check(edges, scores, keys, h2, what=""):
    """Node keys equal, h2 within GAMMA of its scale, scores within the SPEC §6 bound. Returns max error/scale."""
    nodes, h2_ref, ref, scale = gnn_ref.run(edges, with_scale=True)
    assert np.array_equal(keys, nodes), what
    assert np.all(np.isfinite(h2)) and np.all(np.isfinite(scores)), what
    rel = np.abs(h2.astype(np.float64) - h2_ref) / scale
    worst = float(rel.max()) if rel.size else 0.0
    if worst > GAMMA:
        v, j = np.unravel_index(int(rel.argmax()), rel.shape)
        raise AssertionError(f"{what}: h2 error {worst:.3g} x scale > {GAMMA:.3g} at node {v} (key {int(nodes[v]):#x}) "
                             f"col {j}: {h2[v, j]!r} vs {h2_ref[v, j]!r}")
    err = np.abs(scores.astype(np.float64) - ref)
    ok = err <= ATOL + RTOL * np.abs(ref)
    assert ok.all(), (what, float(err.max()), int(err.argmax()), int((~ok).sum()))
    return worst


def score_graph(g, check_oracle=True):
    """Tables + records of g through a fresh handle: (flushed edges, scores, node keys, h2)."""
    b = gg.Built(g)
    h = gg.handle_for(b)
    gg.load(h, b)
    edges = gg.ingest(h, b, check=check_oracle)
    scores, keys, h2 = gg.gnn(h, len(edges))
    h.close()
    return edges, scores, keys, h2


def _events(n_edges, seed, max_count=3):
    """1..max_count events per edge: lognormal durations, 1 in 8 with status 500."""
    rng = np.random.default_rng(seed)
    cnt = 1 + np.arange(n_edges) % max_count
    ee = np.repeat(np.arange(n_edges), cnt)
    dur = np.exp(rng.normal(np.log(2e6), 1.0, len(ee))).astype(np.uint64)
    status = np.where(rng.random(len(ee)) < 0.125, 500, 200)
    return ee, dur, status


def pod_graph(src, dst, seed, rev_every=5):
    """Pods only (pod id = node index when every id below n appears): src[i] -> dst[i], every rev_every-th edge
    ingested as a reversed AMQP row."""
    src, dst = np.asarray(src), np.asarray(dst)
    n = len(src)
    ee, dur, status = _events(n, seed)
    z = np.zeros(n, np.uint8)
    return gg.Graph(z, src, z, dst, ee, dur, status, rev=(np.arange(n) % rev_every) == 1)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- synthetic topologies (alaz_b200/synth) -------------------------------------------------------------------

def _run_synth(S, N, mix, seed, max_pairs=1 << 17):
    t = ol.Topo(S, seed=seed, mix=mix)
    h = capi.Handle(max_endpoints=4 * S, max_pairs=max_pairs)
    h.load_tables(t.pod_ip, t.svc_ip)
    step = 8_000_000
    for i in range(0, N, step):
        h.submit(t.events(i, min(step, N - i)))
    edges = h.flush()
    scores, keys, h2 = gg.gnn(h, len(edges))
    h.close()
    return edges, scores, keys, h2


# The three tests below keep their names for the wgmma layer; each has a twin for the FFMA layer.
SYNTH = [(200, 300_000, abi.MIX_ALL), (2000, 2_000_000, abi.MIX_SURVEY)]


def _synth_scores(S, N, mix):
    edges, scores, keys, h2 = _run_synth(S, N, mix, seed=1000 + S)
    check(edges, scores, keys, h2, f"synth S={S}")
    assert scores.std() > 1e-4    # not a constant


@pytest.mark.parametrize("S,N,mix", SYNTH)
def test_gnn_scores_match_float64_reference(monkeypatch, S, N, mix):
    use_path(monkeypatch, "tc")
    _synth_scores(S, N, mix)


@pytest.mark.parametrize("S,N,mix", SYNTH)
def test_gnn_scores_match_float64_reference_simt_layer(monkeypatch, S, N, mix):
    use_path(monkeypatch, "simt")
    _synth_scores(S, N, mix)


def _config3():
    edges, scores, keys, h2 = _run_synth(50_000, 40_000_000, abi.MIX_SURVEY, seed=77, max_pairs=1 << 21)
    assert len(edges) > 500_000, len(edges)
    check(edges, scores, keys, h2, "config 3")


def test_gnn_at_config3_scale(monkeypatch):
    """BASELINE.json configs[2] names a 50k-service graph: most of a million edges, several hundred thousand nodes.
    The tensor-core layer runs thousands of 128-row tiles with gathers that miss L2; same tolerance."""
    use_path(monkeypatch, "tc")
    _config3()


def test_gnn_at_config3_scale_simt_layer(monkeypatch):
    use_path(monkeypatch, "simt")
    _config3()


def _empty_window_and_quantiles():
    h = capi.Handle(max_endpoints=64, max_pairs=256)
    h.commit()
    assert len(h.flush()) == 0
    n = C.c_size_t(7)
    h._ck(h.L.alz_gnn_score(h.h, None, 0, C.byref(n)), "alz_gnn_score")
    assert n.value == 0
    e = np.zeros(1, dtype=abi.EDGE_OUT)
    e["hist"][0][4] = 10
    e["hist"][0][5] = 10
    qs = np.array([0.25, 0.5, 0.75, 0.99, 1.0])
    out = np.zeros(5)
    assert h.L.alz_edge_quantiles(e.ctypes.data_as(C.c_void_p), qs.ctypes.data_as(C.c_void_p), 5,
                                  out.ctypes.data_as(C.c_void_p)) == 0
    ref = np.array([ol.quantile(e["hist"][0], q) for q in qs])
    assert np.allclose(out, ref, rtol=1e-12)
    h.close()


def test_gnn_on_empty_window_and_quantiles(monkeypatch):
    use_path(monkeypatch, "tc")
    _empty_window_and_quantiles()


def test_gnn_on_empty_window_and_quantiles_simt_layer(monkeypatch):
    use_path(monkeypatch, "simt")
    _empty_window_and_quantiles()


# ---- node counts around the 128-node tile and the one-CTA-per-SM wave -------------------------------------------

def _ring(n, seed):
    """n pods: ring i -> i+1 plus chords i -> 3i+7 (mod n); n = 1 is a single self-loop."""
    pairs = {(i, (i + 1) % n) for i in range(n)} | {(i, (3 * i + 7) % n) for i in range(n) if (3 * i + 7) % n != i}
    src, dst = zip(*sorted(pairs))
    return pod_graph(src, dst, seed)


NODE_COUNTS = {str(k): (lambda s, k=k: k) for k in (1, 2, 15, 16, 17, 127, 128, 129)}
NODE_COUNTS.update({"SMs*128-1": lambda s: s * 128 - 1, "SMs*128": lambda s: s * 128,
                    "SMs*128+1": lambda s: s * 128 + 1, "2*SMs*128+5": lambda s: 2 * s * 128 + 5})


@pytest.mark.parametrize("count", list(NODE_COUNTS))
def test_node_counts_around_tiles_and_waves(path, count):
    """Partial tiles, exactly one wave of one tile per SM, one tile past the wave, and a second lap."""
    n = NODE_COUNTS[count](sm_count())
    edges, scores, keys, h2 = score_graph(_ring(n, seed=n))
    assert len(keys) == n
    check(edges, scores, keys, h2, f"ring n={n}")


# ---- in-degree patterns inside a warp's 16 rows (TMA ring of 8 rows, rows cut at chunk boundaries) ---------------

WARP_PATTERNS = {
    "all_zero": [0] * 16,
    "around_ring_chunks": [7, 8, 9, 16, 17, 7, 8, 9, 16, 17, 8, 16, 24, 1, 9, 17],
    "fifteen_zero_then_50": [0] * 15 + [50],
    "alternating_0_33": [0, 33] * 8,
}
N_PATTERN = 8 * 128 + 37          # eight full tiles and a partial one


def _degree_graph(indeg, seed):
    """Pods 0..n-1, node v with indeg[v] distinct in-neighbours taken cyclically over all nodes (so every node is
    some node's source when sum(indeg) >= n)."""
    n = len(indeg)
    src, dst = [], []
    p = 0
    for v in range(n):
        k = 0
        while k < indeg[v]:
            if p % n != v:
                src.append(p % n); dst.append(v); k += 1
            p += 1
    assert p >= n, "some node would be isolated"
    return pod_graph(src, dst, seed)


@pytest.mark.parametrize("pattern", list(WARP_PATTERNS) + ["one_1000_mid_tile"])
def test_in_degree_patterns_within_a_warp(path, pattern):
    """Even warps of every tile get the pattern, odd warps 5 in-edges per row; or every row 5 and one row of 1000
    in the middle of the second tile."""
    if pattern == "one_1000_mid_tile":
        indeg = np.full(N_PATTERN, 5)
        indeg[128 + 67] = 1000
    else:
        warp_rows = np.arange(N_PATTERN) // 16
        indeg = np.where(warp_rows % 2 == 0, np.array(WARP_PATTERNS[pattern])[np.arange(N_PATTERN) % 16], 5)
    edges, scores, keys, h2 = score_graph(_degree_graph(indeg, seed=len(pattern)))
    assert len(keys) == N_PATTERN
    nodes, u, v, deg, _ = gnn_ref._graph(edges)
    assert np.array_equal(deg, indeg)
    check(edges, scores, keys, h2, pattern)


def test_perfect_matching_most_tiles_per_edge(path):
    n_e = 200_000
    edges, scores, keys, h2 = score_graph(pod_graph(2 * np.arange(n_e), 2 * np.arange(n_e) + 1, seed=3))
    assert len(keys) == 2 * n_e
    check(edges, scores, keys, h2, "matching")


# ---- hubs: one warp sums every in-neighbour row of a hub --------------------------------------------------------

def _star(n_clients, count, dur):
    """Identical pods 1..n -> service 0: rounding errors of the hub's neighbour sum all point the same way."""
    c = np.arange(1, n_clients + 1)
    return gg.Graph.uniform(np.full(n_clients, gg.POD), c, np.full(n_clients, gg.SVC), np.zeros(n_clients, np.int64),
                            dur=dur, count=count)


@pytest.mark.parametrize("n_clients,count,dur", [(100_000, 3, 1_500_000), (1_000_000, 1, 2_000_000)])
def test_hub_of_identical_clients(path, n_clients, count, dur):
    edges, scores, keys, h2 = score_graph(_star(n_clients, count, dur))
    check(edges, scores, keys, h2, f"star {n_clients}")


def test_hub_fed_back_through_its_clients(path):
    """Pod 0 -> pods 1..K and pods 1..K -> pod 0: layer 2 of the hub means K rows that each mean the hub's layer-1
    row."""
    K = 100_000
    c = np.arange(1, K + 1)
    src = np.concatenate([np.zeros(K, np.int64), c])
    dst = np.concatenate([c, np.zeros(K, np.int64)])
    z = np.zeros(2 * K, np.uint8)
    edges, scores, keys, h2 = score_graph(gg.Graph.uniform(z, src, z, dst, dur=3_000_000, count=2))
    check(edges, scores, keys, h2, "hub fed back")


# ---- node sums wrap mod 2^64 ------------------------------------------------------------------------------------

def test_node_latency_sums_wrap_mod_2_64(path):
    """A pod whose two out-edges each carry one event of 2^64-1 ns: its out-latency sum is 2^64-2 (mod 2^64, SPEC
    §6), not 2^65-2; the services' in-sums wrap the same way."""
    M = (1 << 64) - 1
    P, S = gg.POD, gg.SVC
    g = gg.Graph.from_list([
        ((P, 0), (S, 0), [(M, 200)]),
        ((P, 0), (S, 1), [(M, 500)]),
        ((P, 1), (S, 0), [(M, 200), (5_000_000, 200)]),
        ((P, 1), (S, 1), [(3_000_000, 200)]),
        ((P, 2), (S, 1), [(M, 200), (M, 200), (M, 200)]),
    ])
    edges, scores, keys, h2 = score_graph(g)
    # the wrap moves pod 0's mean latency feature by log(2): a reference that did not wrap could not pass
    wrapped = float((2 * M) & M) / 2
    assert abs(np.log1p(wrapped) - np.log1p(2.0 * M / 2)) > 0.5
    check(edges, scores, keys, h2, "latency wrap")


# ---- histogram edges of the quantile scan (lane l owns buckets 2l and 2l+1) -------------------------------------

def _dur_in(b):
    """A duration in bucket b (SPEC §4)."""
    return 100 if b == 0 else (1 << 40) if b == 63 else int(gnn_ref.bucket_lo(b))


HIST_CASES = {
    "p50_tie_end_of_bucket_5_gap": {5: 2, 9: 2},
    "p50_tie_across_lanes_3_4": {3: 3, 4: 3},
    "p50_tie_across_lanes_gap": {7: 5, 12: 5},
    "p50_tie_end_of_bucket_0": {0: 1, 5: 1},
    "p99_tie_end_of_bucket_10": {10: 99, 20: 1},
    "p99_tie_across_lanes": {11: 198, 14: 2},
    "p99_tie_last_lane": {61: 297, 63: 3},
    "all_in_bucket_0": {0: 5},
    "all_in_bucket_63": {63: 4},
    "single_event": {17: 1},
    "first_and_last": {0: 1, 63: 1},
}


def test_histogram_edges_of_the_quantile_scan(path):
    """One edge per case (pod i -> service i % 3); every case's p50 or p99 target lands exactly on a bucket's end
    (with the next non-empty bucket further on, so `>=` and `>` differ), across the 2l+1 | 2l+2 lane boundary,
    or all mass in bucket 0 or 63; 5xx rates 0 and 1 on the extra edges."""
    items = []
    for i, (name, cells) in enumerate(HIST_CASES.items()):
        evs = []
        for b, c in cells.items():
            d = _dur_in(b)
            evs += [((1 << 64) - 1 if b == 63 and k % 2 else d, 200) for k in range(c)]
        items.append(((gg.POD, i), (gg.SVC, i % 3), evs))
    k = len(items)
    items.append(((gg.POD, k), (gg.SVC, 0), [(3_000_000, 500)] * 4))            # 5xx rate 1
    items.append(((gg.POD, k), (gg.SVC, 1), [(3_000_000, 200)] * 4))            # 5xx rate 0
    items.append(((gg.POD, k + 1), (gg.OUT, 0xFFFFFFFF), [(999, 503), (1000, 599)]))
    edges, scores, keys, h2 = score_graph(gg.Graph.from_list(items))
    names = list(HIST_CASES)
    for e in edges[(edges["from_type"] == gg.POD) & (edges["from"] < len(names))]:
        name = names[int(e["from"])]
        assert {b: int(c) for b, c in enumerate(e["hist"]) if c} == HIST_CASES[name], name
    check(edges, scores, keys, h2, "histogram edges")


# ---- every node kind, self-loops, reversed rows: hypothesis -----------------------------------------------------

POD_IDS = [0, 1, 2, 3, 5, 8, 13, 100, 4097, (1 << 29) - 1]
SVC_IDS = [0, 1, 7, (1 << 29) - 1]
OUT_ADDRS = [1, abi.ip("8.8.8.8"), abi.ip("203.0.113.7"), 0xFFFFFFFE, 0xFFFFFFFF]
HOST_IDS = [0, 1, 99, 123456789, 0xFFFFFFFF]
DURS = [0, 255, 256, 383, 384, (1 << 40) - 1, 1 << 40, (1 << 64) - 1]
KINDS = ["pp", "pp_rev", "ps", "po", "ph", "sp", "op"]

dur_s = st.one_of(st.sampled_from(DURS), st.floats(-4, 4).map(lambda x: int(2e6 * np.exp(x))))
ev_s = st.tuples(dur_s, st.sampled_from([200, 404, 500, 503, 599, 600]))
edge_s = st.tuples(st.sampled_from(KINDS), st.integers(0, 200), st.integers(0, 200),
                   st.lists(ev_s, min_size=1, max_size=4))


def _hyp_graph(raw, n_pods, n_svcs):
    pods = sorted(set(POD_IDS) | set(range(20, 20 + n_pods)))
    svcs = sorted(set(SVC_IDS) | set(range(10, 10 + n_svcs)))
    P, S, O, H = gg.POD, gg.SVC, gg.OUT, gg.HOST
    ends = {}
    for kind, i, j, evs in raw:
        p, q = pods[i % len(pods)], pods[j % len(pods)]
        a, b, rev = {
            "pp": ((P, p), (P, q), False), "pp_rev": ((P, p), (P, q), True), "ps": ((P, p), (S, svcs[j % len(svcs)]), False),
            "po": ((P, p), (O, OUT_ADDRS[j % 5]), False), "ph": ((P, p), (H, HOST_IDS[j % 5]), False),
            "sp": ((S, svcs[i % len(svcs)]), (P, q), False), "op": ((O, OUT_ADDRS[i % 5]), (P, q), False),
        }[kind]
        if (a, b) in ends:
            ends[(a, b)][1].extend(evs)
        else:
            ends[(a, b)] = (rev, list(evs))
    return gg.Graph.from_list([(a, b, evs, rev) for (a, b), (rev, evs) in ends.items()])


_hyp_state = {}


@settings(max_examples=40, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(raw=st.lists(edge_s, min_size=1, max_size=150), n_pods=st.integers(0, 150), n_svcs=st.integers(0, 40))
def test_small_graphs_of_every_kind(path, raw, n_pods, n_svcs):
    """One handle per layer path, reused: every example rewrites the tables and flushes its own window."""
    g = _hyp_graph(raw, n_pods, n_svcs)
    b = gg.Built(g)
    if path not in _hyp_state:
        _hyp_state[path] = (capi.Handle(max_endpoints=512, max_pairs=1024), {})
    h, cur = _hyp_state[path]
    for table, ips in cur.items():
        for ip in ips:
            h.erase(table, ip)
    cur[abi.TABLE_POD] = b.pod_ip.tolist()
    cur[abi.TABLE_SVC] = b.svc_ip.tolist()
    gg.load(h, b)
    edges = gg.ingest(h, b)
    scores, keys, h2 = gg.gnn(h, len(edges))
    assert len(keys) <= 300
    check(edges, scores, keys, h2, "hypothesis")


# ---- determinism -------------------------------------------------------------------------------------------------

def _mixed_graph():
    """Degrees 0..40 and a hub of 3000, pods plus a service, an outbound and a host-keyed node."""
    n = 3 * 128 + 21
    indeg = (np.arange(n) * 7) % 41
    indeg[200] = 0
    g = _degree_graph(indeg, seed=11)
    hub = 3000
    u8, u64 = np.uint8, np.uint64
    ft = np.concatenate([g.ft, np.zeros(hub + 2, u8)])
    fv = np.concatenate([g.fv, np.arange(hub, dtype=u64), np.array([1, 2], u64)])
    tt = np.concatenate([g.tt, np.full(hub, gg.SVC, u8), np.array([gg.OUT, gg.HOST], u8)])
    tv = np.concatenate([g.tv, np.full(hub, 5, u64), np.array([0xFFFFFFFF, 0xFFFFFFFF], u64)])
    ee, dur, status = _events(len(ft), seed=12)
    return gg.Graph(ft, fv, tt, tv, ee, dur, status, rev=np.concatenate([g.rev, np.zeros(hub + 2, bool)]))


def test_scores_are_deterministic(path):
    """Two alz_gnn_score calls on one window, alz_gnn_score_device, and the same graph submitted in another
    event order on a fresh handle: bitwise-identical scores."""
    b = gg.Built(_mixed_graph())
    h = gg.handle_for(b)
    gg.load(h, b)
    edges = gg.ingest(h, b)
    s1, keys, h2 = gg.gnn(h, len(edges))
    s2, _, _ = gg.gnn(h, len(edges))
    s3 = gg.gnn_device(h, len(edges))
    h.close()
    check(edges, s1, keys, h2, "determinism")
    assert s1.tobytes() == s2.tobytes()
    assert s1.tobytes() == s3.tobytes()
    h = gg.handle_for(b)
    gg.load(h, b)
    edges2 = gg.ingest(h, b, order=np.random.default_rng(9).permutation(len(b.recs)), check=False)
    assert edges2.tobytes() == edges.tobytes()
    s4, _, _ = gg.gnn(h, len(edges))
    h.close()
    assert s1.tobytes() == s4.tobytes()
