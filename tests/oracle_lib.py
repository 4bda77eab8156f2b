"""ctypes wrapper over oracle/_build/liboracle.so (CPU oracle + host synth).

Test infrastructure: imported by tests/, bench.py (cpu_baseline / --impl
reference) and __graft_entry__.smoke() only. The product never imports this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from alaz_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(ROOT, "oracle", "_build", "liboracle.so")


def build(force=False):
    src = [os.path.join(ROOT, "oracle", "alz_oracle.c"), os.path.join(ROOT, "oracle", "alz_fastcpu.c"),
           os.path.join(ROOT, "oracle", "alz_oracle.h"),
           os.path.join(ROOT, "alaz_b200", "synth", "alz_synth_topo.c"),
           os.path.join(ROOT, "alaz_b200", "synth", "alz_synth.h"),
           os.path.join(ROOT, "include", "alazgpu.h")]
    if not force and os.path.exists(LIB_PATH):
        t = os.path.getmtime(LIB_PATH)
        if all(os.path.getmtime(s) <= t for s in src):
            return LIB_PATH
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")],
                          stdout=subprocess.DEVNULL)
    return LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(LIB_PATH)
        vp, u32, u64, sz = C.c_void_p, C.c_uint32, C.c_uint64, C.c_size_t
        L.orc_create.restype = vp
        L.orc_destroy.argtypes = [vp]
        L.orc_table_upsert.argtypes = [vp, C.c_int, u32, u32]
        L.orc_table_erase.argtypes = [vp, C.c_int, u32]
        L.orc_process_l7.argtypes = [vp, vp, sz, C.c_int]
        L.orc_process_l7_hosts.argtypes = [vp, vp, sz, vp, C.POINTER(C.c_char_p), sz]
        L.orc_parse_http_host.argtypes = [C.c_char_p, sz, C.c_char_p, sz]
        L.orc_parse_http_host.restype = sz
        L.orc_epoch.argtypes = [u64, u64, u64, u64]
        L.orc_epoch.restype = u64
        L.orc_edges.argtypes = [vp, vp, sz]
        L.orc_edges.restype = sz
        L.orc_window_reset.argtypes = [vp]
        L.orc_stats.argtypes = [vp, C.POINTER(abi.Stats)]
        L.orc_bucket.argtypes = [u64]
        L.orc_bucket.restype = u32
        L.orc_quantile.argtypes = [vp, C.c_double]
        L.orc_quantile.restype = C.c_double
        L.orc_compact_raw.argtypes = [vp, sz, vp]
        L.orc_sockline_create.restype = vp
        L.orc_sockline_destroy.argtypes = [vp]
        L.orc_sockline_add.argtypes = [vp, u64, vp]
        L.orc_sockline_get.argtypes = [vp, u64, vp]
        L.orc_sockline_get.restype = C.c_int
        L.orc_sockline_len.argtypes = [vp]
        L.orc_sockline_len.restype = sz
        L.orc_sockmaps_create.restype = vp
        L.orc_sockmaps_destroy.argtypes = [vp]
        L.orc_sockmaps_process_tcp.argtypes = [vp, vp, sz, C.POINTER(u64)]
        L.orc_sockmaps_lookup.argtypes = [vp, vp, sz, vp]
        L.orc_sockmaps_lookup_at.argtypes = [vp, vp, sz, u64, vp]
        L.orc_sockmaps_gc.argtypes = [vp]
        L.orc_sockmaps_records.argtypes = [vp]
        L.orc_sockmaps_records.restype = sz
        L.orc_sockmaps_lines.argtypes = [vp, vp, vp, vp, sz]
        L.orc_sockmaps_lines.restype = sz
        L.orc_sockmaps_join.argtypes = [vp, vp, vp, sz, u64, C.POINTER(u64)]
        L.orc_sockmaps_alive.argtypes = [vp, vp, vp, sz]
        L.orc_sockmaps_alive.restype = sz
        L.orc_sockline_get_at.argtypes = [vp, u64, u64, vp]
        L.orc_sockline_get_at.restype = C.c_int
        L.orc_sockline_delete_unused.argtypes = [vp]
        L.orc_fast_create.argtypes = [u32]
        L.orc_fast_create.restype = vp
        L.orc_fast_destroy.argtypes = [vp]
        L.orc_fast_table_upsert.argtypes = [vp, C.c_int, u32, u32]
        L.orc_fast_process.argtypes = [vp, vp, sz, C.c_int]
        L.orc_fast_edges.argtypes = [vp, vp, sz]
        L.orc_fast_edges.restype = sz
        L.orc_fast_reset.argtypes = [vp]
        L.orc_fast_stats.argtypes = [vp, C.POINTER(abi.Stats)]
        L.alz_synth_topo_create.argtypes = [u32, u64, u32]
        L.alz_synth_topo_create.restype = C.POINTER(abi.SynthTopo)
        L.alz_synth_topo_destroy.argtypes = [C.POINTER(abi.SynthTopo)]
        L.alz_synth_fill.argtypes = [C.POINTER(abi.SynthTopo), u64, u64, vp]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class Oracle:
    """The reference aggregator's resolve/emit path, restated (oracle/alz_oracle.c)."""

    def __init__(self):
        self.L = lib()
        self.h = self.L.orc_create()

    def close(self):
        if self.h:
            self.L.orc_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def upsert(self, table, ip, id_):
        self.L.orc_table_upsert(self.h, table, int(ip), int(id_))

    def erase(self, table, ip):
        self.L.orc_table_erase(self.h, table, int(ip))

    def load_tables(self, pod_ip, svc_ip):
        for k, v in enumerate(pod_ip):
            self.upsert(abi.TABLE_POD, int(v), k)
        for k, v in enumerate(svc_ip):
            self.upsert(abi.TABLE_SVC, int(v), k)

    def process(self, recs, nthreads=1):
        recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
        self.L.orc_process_l7(self.h, _ptr(recs), len(recs), nthreads)

    def process_hosts(self, recs, host_idx, names):
        """Events with their HTTP Host header: host_idx[i] = 0 (none) or 1 + index into names."""
        recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
        host_idx = np.ascontiguousarray(host_idx, dtype=np.uint32)
        self._names = (C.c_char_p * max(1, len(names)))(*[n.encode() for n in names])   # must outlive edges()
        self.L.orc_process_l7_hosts(self.h, _ptr(recs), len(recs), _ptr(host_idx), self._names, len(names))

    def edges(self):
        n = self.L.orc_edges(self.h, None, 0)
        out = np.zeros(n, dtype=abi.EDGE_OUT)
        if n:
            self.L.orc_edges(self.h, _ptr(out), n)
        return out

    def reset_window(self):
        self.L.orc_window_reset(self.h)

    def stats(self):
        st = abi.Stats()
        self.L.orc_stats(self.h, C.byref(st))
        return st.as_dict()


class FastCpu:
    """The "fair" CPU arm (oracle/alz_fastcpu.c): integer keys, flat tables, per-thread accumulators."""

    def __init__(self, max_endpoints=1 << 16):
        self.L = lib()
        self.h = self.L.orc_fast_create(int(max_endpoints))

    def close(self):
        if self.h:
            self.L.orc_fast_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def load_tables(self, pod_ip, svc_ip):
        for k, v in enumerate(pod_ip):
            self.L.orc_fast_table_upsert(self.h, abi.TABLE_POD, int(v), k)
        for k, v in enumerate(svc_ip):
            self.L.orc_fast_table_upsert(self.h, abi.TABLE_SVC, int(v), k)

    def upsert(self, table, ip, id_):
        self.L.orc_fast_table_upsert(self.h, table, int(ip), int(id_))

    def process(self, recs, nthreads=1):
        recs = np.ascontiguousarray(recs, dtype=abi.L7_REC)
        self.L.orc_fast_process(self.h, _ptr(recs), len(recs), nthreads)

    def edges(self):
        n = self.L.orc_fast_edges(self.h, None, 0)
        out = np.zeros(n, dtype=abi.EDGE_OUT)
        if n:
            self.L.orc_fast_edges(self.h, _ptr(out), n)
        return out

    def reset_window(self):
        self.L.orc_fast_reset(self.h)

    def stats(self):
        st = abi.Stats()
        self.L.orc_fast_stats(self.h, C.byref(st))
        return st.as_dict()


def parse_http_host(payload: bytes) -> str:
    out = C.create_string_buffer(1100)
    lib().orc_parse_http_host(payload, len(payload), out, len(out))
    return out.value.decode()


def epoch(first_kernel, first_user, window_ns, write_time):
    return int(lib().orc_epoch(int(first_kernel), int(first_user), int(window_ns), int(write_time)))


def bucket(d):
    return int(lib().orc_bucket(int(d)))


def quantile(hist, q):
    h = np.ascontiguousarray(hist, dtype=np.uint32)
    return float(lib().orc_quantile(_ptr(h), float(q)))


def compact_raw(raw):
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    n = raw.size // abi.BPF_L7_EVENT_SIZE
    out = np.zeros(n, dtype=abi.L7_REC)
    lib().orc_compact_raw(_ptr(raw), n, _ptr(out))
    return out


class Topo:
    """Synthetic cluster + stream tables (alaz_b200/synth/alz_synth_topo.c), host side."""

    def __init__(self, n_services, seed=0xA1A20000, mix=abi.MIX_SURVEY):
        self.L = lib()
        self.p = self.L.alz_synth_topo_create(n_services, seed, mix)
        if not self.p:
            raise MemoryError("alz_synth_topo_create failed")
        t = self.p.contents
        self.n_services, self.n_pods = t.n_services, t.n_pods
        self.n_edges, self.n_outbound = t.n_edges, t.n_outbound
        self.pod_ip = np.ctypeslib.as_array(t.pod_ip, (t.n_pods,)).copy()
        self.svc_ip = np.ctypeslib.as_array(t.svc_ip, (t.n_services,)).copy()
        self.out_ip = np.ctypeslib.as_array(t.out_ip, (t.n_outbound,)).copy()

    def arrays(self):
        """Copies of the sampling tables (for upload to the device generator)."""
        t = self.p.contents
        E = t.n_edges
        return dict(
            edge_saddr=np.ctypeslib.as_array(t.edge_saddr, (E,)).copy(),
            edge_daddr=np.ctypeslib.as_array(t.edge_daddr, (E,)).copy(),
            edge_flags=np.ctypeslib.as_array(t.edge_flags, (E,)).copy(),
            alias_thresh=np.ctypeslib.as_array(t.alias_thresh, (E,)).copy(),
            alias_idx=np.ctypeslib.as_array(t.alias_idx, (E,)).copy(),
            lat_q=np.ctypeslib.as_array(t.lat_q, (4097,)).copy(),
        )

    def view(self):
        return self.p.contents.view

    def events(self, first, n):
        out = np.zeros(n, dtype=abi.L7_REC)
        self.L.alz_synth_fill(self.p, int(first), int(n), _ptr(out))
        return out

    def close(self):
        if self.p:
            self.L.alz_synth_topo_destroy(self.p)
            self.p = None

    def __del__(self):
        self.close()


class SockMaps:
    """processTcpConnect + SocketLine lookups, restated (oracle/alz_oracle.c)."""

    def __init__(self):
        self.L = lib()
        self.h = self.L.orc_sockmaps_create()
        self.localhost_dropped = 0

    def process(self, recs):
        recs = np.ascontiguousarray(recs, dtype=abi.TCP_REC)
        d = C.c_uint64(0)
        self.L.orc_sockmaps_process_tcp(self.h, _ptr(recs), len(recs), C.byref(d))
        self.localhost_dropped += d.value

    def lookup(self, q, now_ns=1):
        q = np.ascontiguousarray(q, dtype=abi.SOCK_QUERY)
        out = np.zeros(len(q), dtype=abi.SOCK_RESULT)
        self.L.orc_sockmaps_lookup_at(self.h, _ptr(q), len(q), int(now_ns), _ptr(out))
        return out

    def gc(self):
        self.L.orc_sockmaps_gc(self.h)

    def records(self):
        return int(self.L.orc_sockmaps_records(self.h))

    def lines(self):
        """{(pid, fd): number of values} of every line, including lines emptied by the GC."""
        n = int(self.L.orc_sockmaps_lines(self.h, None, None, None, 0))
        pid, fd, ln = np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(n, np.uint64)
        if n:
            self.L.orc_sockmaps_lines(self.h, _ptr(pid), _ptr(fd), _ptr(ln), n)
        return {(int(p), int(f)): int(k) for p, f, k in zip(pid, fd, ln)}

    def join(self, recs, keys, now_ns=1):
        """recs with empty 5-tuples filled from the timelines (a copy) and the number filled."""
        recs = np.ascontiguousarray(recs, dtype=abi.L7_REC).copy()
        keys = np.ascontiguousarray(keys, dtype=abi.SOCK_QUERY)
        j = C.c_uint64(0)
        self.L.orc_sockmaps_join(self.h, _ptr(recs), _ptr(keys), len(recs), int(now_ns), C.byref(j))
        return recs, j.value

    def alive(self, oracle, cap=1 << 20):
        out = np.zeros(cap, dtype=abi.ALIVE_CONN)
        n = self.L.orc_sockmaps_alive(self.h, oracle.h, _ptr(out), cap)
        return out[:n]

    def close(self):
        if self.h:
            self.L.orc_sockmaps_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()
