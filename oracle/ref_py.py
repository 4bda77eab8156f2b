"""Second, independent restatement of the reference resolve/emit path in plain
Python (dicts and strings, small cases only). TEST INFRASTRUCTURE ONLY.

It exists to cross-check oracle/alz_oracle.c on random small cases and against
the hand-derived golden vectors; it shares no code with the C oracle or with
the product. PARITY UNPINNED for resolve/emit (see oracle/alz_oracle.h).
"""

# ebpf/l7_req/l7.go:48-71
_PROTO = {0: "UNKNOWN", 1: "HTTP", 2: "AMQP", 3: "POSTGRES", 4: "HTTP2",
          5: "REDIS", 6: "KAFKA", 7: "MYSQL", 8: "MONGO"}
# ebpf/l7_req/l7.go:204-325, switch at :712-734
_METHOD = {
    "HTTP": {1: "GET", 2: "POST", 3: "PUT", 4: "PATCH", 5: "DELETE", 6: "HEAD",
             7: "CONNECT", 8: "OPTIONS", 9: "TRACE"},
    "AMQP": {1: "PUBLISH", 2: "DELIVER"},
    "POSTGRES": {1: "CLOSE_OR_TERMINATE", 2: "SIMPLE_QUERY", 3: "EXTENDED_QUERY"},
    "HTTP2": {1: "CLIENT_FRAME", 2: "SERVER_FRAME"},
    "REDIS": {1: "COMMAND", 2: "PUSHED_EVENT", 3: "PING"},
    "KAFKA": {1: "PRODUCE_REQUEST", 2: "FETCH_RESPONSE"},
    "MYSQL": {1: "TEXT_QUERY", 2: "PREPARE_STMT", 3: "EXEC_STMT", 4: "STMT_CLOSE"},
}
NB = 64


def ip_string(x):  # IntToIPv4(x).String(), aggregator/data.go:1751-1767
    return "%d.%d.%d.%d" % ((x >> 24) & 255, (x >> 16) & 255, (x >> 8) & 255, x & 255)


def bucket(d):  # docs/SPEC.md §4
    if d < 256:
        return 0
    o = d.bit_length() - 1
    if o >= 40:
        return NB - 1
    return 2 * (o - 8) + ((d >> (o - 1)) & 1)


def parse_http_payload_host(request):  # parseHttpPayload's hostHeader, aggregator/data.go:508-531
    if isinstance(request, bytes):
        request = request.decode("latin-1")
    lines = request.split("\n")
    host = ""
    for line in lines[1:]:
        if line.startswith("Host:"):
            parts = line.split(" ")
            if len(parts) >= 2:
                host = parts[1]
                if host.endswith("\r"):
                    host = host[:-1]
                break
    return host


class Aggregator:
    def __init__(self):
        self.pod_ip_to_uid = {}   # cluster.go:15
        self.svc_ip_to_uid = {}   # cluster.go:16
        self.groups = {}
        self.stats = dict(events_in=0, rows_emitted=0, not_request=0, src_unresolved=0)

    def set_from_to_v2(self, row, host_header=""):  # aggregator/data.go:827-870
        uid = self.pod_ip_to_uid.get(row["FromIP"])
        if uid is None:
            return False
        row["FromUID"], row["FromType"] = uid, "pod"
        s = self.svc_ip_to_uid.get(row["ToIP"])
        if s is not None:
            row["ToUID"], row["ToType"] = s, "service"
            return True
        p = self.pod_ip_to_uid.get(row["ToIP"])
        if p is not None:
            row["ToUID"], row["ToType"] = p, "pod"
            return True
        if host_header != "":
            row["ToUID"], row["ToType"] = host_header, "outbound"  # :851-854
            return True
        row["ToUID"], row["ToType"] = row["ToIP"], "outbound"  # :862, DNS treated as failing
        return True

    def process_l7(self, rec, payload=None):  # aggregator/data.go:1364-1383; payload: the HTTP request bytes, if any
        self.stats["events_in"] += 1
        proto = _PROTO.get(int(rec["protocol"]), "Unknown")
        mf = int(rec["method_flags"])
        method = _METHOD.get(proto, {}).get(mf & 0x3F, "Unknown")
        tls, reject = bool(mf & 0x80), bool(mf & 0x40)
        if proto not in ("HTTP", "AMQP", "REDIS", "POSTGRES", "MYSQL", "MONGO"):
            self.stats["not_request"] += 1
            return
        if proto in ("POSTGRES", "MYSQL", "MONGO") and reject:
            self.stats["not_request"] += 1
            return
        row = dict(Latency=int(rec["duration_ns"]), FromIP=ip_string(int(rec["saddr"])),
                   ToIP=ip_string(int(rec["daddr"])), Protocol=proto, Tls=tls,
                   StatusCode=int(rec["status"]), Method=method)
        host = parse_http_payload_host(payload) if (proto == "HTTP" and payload is not None) else ""   # :1213
        if not self.set_from_to_v2(row, host):
            self.stats["src_unresolved"] += 1
            return
        if (proto == "AMQP" and method == "DELIVER") or (proto == "REDIS" and method == "PUSHED_EVENT"):
            # Request.ReverseDirection, datastore/dto.go:246-251
            row["FromIP"], row["ToIP"] = row["ToIP"], row["FromIP"]
            row["FromUID"], row["ToUID"] = row["ToUID"], row["FromUID"]
            row["FromType"], row["ToType"] = row["ToType"], row["FromType"]
        if proto == "HTTP" and tls:
            row["Protocol"] = "HTTPS"
        self.persist_request(row)

    def persist_request(self, row):
        key = (row["FromType"], row["FromUID"], row["ToType"], row["ToUID"])
        g = self.groups.setdefault(key, dict(count=0, err5xx=0, lat_sum=0, hist=[0] * NB))
        g["count"] += 1
        if row["Protocol"] in ("HTTP", "HTTPS") and 500 <= row["StatusCode"] < 600:
            g["err5xx"] += 1
        g["lat_sum"] += row["Latency"]
        g["hist"][bucket(row["Latency"])] += 1
        self.stats["rows_emitted"] += 1


# ---------------------------------------------------------------------------------------------------------------
# SocketLine (aggregator/sock_num_line.go), restated from the Go source independently of oracle/alz_oracle.c:
# Python lists and bisect instead of the C arrays and hand-written binary searches.
# ---------------------------------------------------------------------------------------------------------------
import bisect  # noqa: E402

ONE_MINUTE_NS = 60 * 10**9
FIVE_MINUTES_NS = 5 * ONE_MINUTE_NS
MASK64 = (1 << 64) - 1


class SocketLine:
    """Values: list of [timestamp, sockinfo-or-None, last_match]; sockinfo = (saddr, daddr, sport, dport)."""

    def __init__(self):
        self.values = []

    def add_value(self, ts, si):  # :62-80, insertIntoSortedSlice :311-322
        if self.values:
            last = self.values[-1]
            if last[1] is not None and si is not None and last[1] == si:
                return
        # sort.Search for the first index with Timestamp >= ts
        idx = bisect.bisect_left([v[0] for v in self.values], ts)
        self.values.insert(idx, [ts, si, 0])

    def get_value(self, ts, now):  # :82-158
        v = self.values
        if not v:
            return None
        index = bisect.bisect_left([x[0] for x in v], ts)      # first i with !(Timestamp < ts)
        if index == len(v):
            v[index - 1][2] = now                                # :96
            if v[-1][1] is None:
                if index - 2 >= 0 and v[index - 2][1] is not None and (ts - v[index - 2][0]) < ONE_MINUTE_NS:
                    return v[index - 2][1]
                return None
            return v[-1][1]
        if index == 0:
            return v[0][1]                                       # an open socket or None (:112-118)
        si = v[index - 1][1]
        if si is None:
            prev = v[index - 2] if index - 2 >= 0 else None
            after = v[index]
            if prev is not None and prev[1] is not None and after[1] is not None:
                if prev[1][1] == after[1][1] and prev[1][3] == after[1][3]:     # Daddr, Dport
                    return prev[1] if ts - prev[0] < after[0] - ts else after[1]
            return None
        v[index - 1][2] = now                                    # :156
        return si

    def delete_unused(self):  # :160-209, as written
        v = self.values
        if len(v) <= 1:
            return
        result = []
        i = 0
        while i < len(v) - 1:
            if v[i][1] is not None and v[i + 1][1] is not None:
                result.append(v[i + 1])
                i += 2
            else:
                result.append(v[i])
                i += 1
        v = result
        last_matched = 0
        for x in reversed(v):
            if x[2] != 0 and x[2] > last_matched:
                last_matched = x[2]
        i = len(v) - 1
        while i >= 1:
            # uint64 in Go: a stamp within five minutes of 2^64 wraps to a small sum
            if v[i][1] is None and v[i - 1][1] is not None and ((v[i - 1][2] + FIVE_MINUTES_NS) & MASK64) < last_matched:
                v = v[:i - 1] + v[i + 1:]
                i -= 1
            i -= 1
        self.values = v


class SocketMaps:
    """processTcpConnect (aggregator/data.go:404-506) over SocketMaps[pid].M[fd], plus findRelatedSocket
    (:1407-1429) and sendOpenConnection (:1628-1679)."""

    def __init__(self):
        self.lines = {}
        self.localhost_dropped = 0

    def process_tcp(self, typ, pid, fd, ts, saddr, daddr, sport, dport):
        if typ not in (1, 5):
            return
        if ip_string(saddr) == "127.0.0.1" or ip_string(daddr) == "127.0.0.1":
            self.localhost_dropped += 1
            return
        if typ == 1:
            self.lines.setdefault((pid, fd), SocketLine()).add_value(ts, (saddr, daddr, sport, dport))
        else:
            ln = self.lines.get((pid, fd))
            if ln is not None:
                ln.add_value(ts, None)

    def lookup(self, pid, fd, ts, now):
        ln = self.lines.get((pid, fd))
        return None if ln is None else ln.get_value(ts, now)

    def gc(self):
        for ln in self.lines.values():
            ln.delete_unused()

    def alive(self, pod_ip_to_uid, svc_ip_to_uid):
        """Rows (from_ip, from_uid, from_port, to_ip, to_type, to_uid, to_port) of sendOpenConnection."""
        out = []
        for ln in self.lines.values():
            if not ln.values:
                continue
            t = ln.values[-1]
            if t[1] is None:
                continue
            saddr, daddr, sport, dport = t[1]
            from_uid = pod_ip_to_uid.get(ip_string(saddr))
            if from_uid is None:
                continue
            to_ip = ip_string(daddr)
            if to_ip in svc_ip_to_uid:
                to_type, to_uid = "service", svc_ip_to_uid[to_ip]
            elif to_ip in pod_ip_to_uid:
                to_type, to_uid = "pod", pod_ip_to_uid[to_ip]
            else:
                to_type, to_uid = "outbound", to_ip
            out.append((saddr, from_uid, sport, daddr, to_type, to_uid, dport))
        return out
