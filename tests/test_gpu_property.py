"""GPU property test (hypothesis): arbitrary small tables and event lists through the C ABI against the
oracle — pod-and-service IPs, 0.0.0.0 / 255.255.255.255 endpoints, every protocol byte, all method/flag
bytes, boundary statuses and durations. One handle is reused: every example rewrites the tables."""
import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st

import oracle_lib as ol
from alaz_b200 import abi, capi
from helpers import edges_equal, explain_diff

pytestmark = pytest.mark.gpu

IPS = [abi.ip("10.0.0.%d" % i) for i in range(1, 9)] + [0, 0xFFFFFFFF, abi.ip("8.8.8.8"), abi.ip("127.0.0.1")]
ip_s = st.sampled_from(IPS)
# protocol bytes: the defined ones and their neighbours, and any byte without ALZ_PROTO_F_HOSTKEY (bit 7 set, or
# 9..63: no protocol, no row)
proto_s = st.one_of(st.integers(0, 12), st.integers(0, 255).map(lambda p: p & ~abi.PROTO_F_HOSTKEY))
event_s = st.tuples(ip_s, ip_s, proto_s, st.integers(0, 255),
                    st.sampled_from([0, 1, 2, 200, 404, 499, 500, 503, 599, 600, 65535]),
                    st.sampled_from([0, 1, 255, 256, 383, 384, 10**6, (1 << 40) - 1, 1 << 40, (1 << 64) - 1]))
table_s = st.dictionaries(ip_s, st.integers(0, 50), max_size=8)

_state = {}


def _handle(flags):
    if flags not in _state:
        _state[flags] = (capi.Handle(max_endpoints=64, max_pairs=512, flags=flags), {}, {})
    return _state[flags]


@pytest.mark.parametrize("flags", [0, abi.CFG_EAGER_JOIN])
@settings(max_examples=60, deadline=None, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(pods=table_s, svcs=table_s, events=st.lists(event_s, max_size=80))
def test_gpu_equals_oracle_on_arbitrary_small_inputs(flags, pods, svcs, events):
    h, cur_pods, cur_svcs = _handle(flags)
    for ip in list(cur_pods):
        h.erase(abi.TABLE_POD, ip)
    for ip in list(cur_svcs):
        h.erase(abi.TABLE_SVC, ip)
    cur_pods.clear(); cur_svcs.clear()
    o = ol.Oracle()
    for ip, i in pods.items():
        h.upsert(abi.TABLE_POD, ip, i); o.upsert(abi.TABLE_POD, ip, i); cur_pods[ip] = i
    for ip, i in svcs.items():
        h.upsert(abi.TABLE_SVC, ip, i); o.upsert(abi.TABLE_SVC, ip, i); cur_svcs[ip] = i
    h.commit()
    recs = np.zeros(len(events), dtype=abi.L7_REC)
    for k, (s, d, proto, mf, status, dur) in enumerate(events):
        recs[k] = (s, d, 1000 + k, 80, status, proto, mf, dur, k)
    before = h.stats()
    h.submit(recs)
    o.process(recs)
    got, exp = h.flush(), o.edges()
    assert edges_equal(got, exp), explain_diff(got, exp)
    after, ost = h.stats(), o.stats()
    for key in ("events_in", "rows_emitted", "not_request", "src_unresolved"):
        assert after[key] - before[key] == ost[key], (key, after[key] - before[key], ost[key])
