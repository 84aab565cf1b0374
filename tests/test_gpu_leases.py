"""DHCP lease census and expiry sweep (bng_dhcp_lease_census / bng_dhcp_lease_sweep): the GPU's records against the
definitions of include/bng_b200.h, restated here in numpy over bng_map_dump of the five DHCP maps.

The definitions, restated:
  - an entry is expired at now_ns when now_ns // 10^9 > lease_expiry, and due when now_ns // 10^9 > lease_expiry +
    grace_s (saturating);
  - one pool record per pool_id that keys ip_pools or is named by a lease entry: unexpired entries per map, expired
    entries, distinct addresses of the unexpired entries, those outside network/prefix_len (addresses in the order the
    context was told, wire bytes or numeric words; all of them without an ip_pools entry, none inside a prefix_len > 32), conflicts (addresses held by two or more
    unexpired entries of the pool within one map), prefix_hosts and permille;
  - the sweep removes the due entries and the circuit_id_map entries whose value MAC keys a removed subscriber_pools
    entry, and nothing else."""
import errno

import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import layouts as L
from bng_b200 import synth as S
from bng_b200.layouts import as_bytes
from oracle import pyoracle

pytestmark = pytest.mark.gpu

LEASE_MAPS = L.LEASE_MAPS
DHCP_MAPS = LEASE_MAPS + ("circuit_id_map", "ip_pools")
POOL_FIELDS = [f for f in L.bng_lease_pool_use.names if f != "pad"]
NOW_S = 1_000_000
NS = 10**9
U64_MAX = 2**64 - 1


def _small(**kw):
    from bng_b200 import Dataplane
    kw.setdefault("max_subscribers", 1 << 12)
    return Dataplane(max_batch=1 << 12, max_nat_sessions=1 << 12, max_eim_mappings=1 << 12, **kw)


def _dumps(dp):
    return {m: dp.dump(m) for m in DHCP_MAPS}


def _pa(v):
    return np.ascontiguousarray(v).view(L.pool_assignment).reshape(-1) if len(v) else np.zeros(0, L.pool_assignment)


def _be(b4, wire=True):
    """The address a 4-byte field means: its bytes in wire order, or a little-endian word holding the numeric value."""
    b = b4.astype(np.int64)
    return b[:, 0] << 24 | b[:, 1] << 16 | b[:, 2] << 8 | b[:, 3] if wire else b[:, 3] << 24 | b[:, 2] << 16 | b[:, 1] << 8 | b[:, 0]


# ---------------------------------------------------------------------------
# the rules, restated
# ---------------------------------------------------------------------------
def census_rule(d, now_ns, wire=True):
    now_s = now_ns // NS
    pk, pv = d["ip_pools"]
    pools = {int(k): v for k, v in zip(np.ascontiguousarray(pk).view("<u4").reshape(-1), _pa_pool(pv))}
    ent = []
    for m, name in enumerate(LEASE_MAPS):
        a = _pa(d[name][1])
        for pool, ip, exp in zip(a["pool_id"].tolist(), _be(a["allocated_ip"], wire).tolist() if len(a) else [], a["lease_expiry"].tolist()):
            ent.append((m, pool, ip, now_s > exp))
    ids = sorted(set(pools) | {e[1] for e in ent})
    recs = np.zeros(len(ids), L.bng_lease_pool_use)
    for r, pid in zip(recs, ids):
        live = [e for e in ent if e[1] == pid and not e[3]]
        for m in range(3):
            r["entries"][m] = sum(1 for e in live if e[0] == m)
        r["expired"] = sum(1 for e in ent if e[1] == pid and e[3])
        addrs = {e[2] for e in live}
        r["addrs"] = len(addrs)
        r["known"] = pid in pools
        hosts = 0
        if pid in pools:
            net, pl = int(_be(pools[pid]["network"][None], wire)[0]), int(pools[pid]["prefix_len"])
            hosts = 0 if pl > 32 else min(1 << (32 - pl), 2**32 - 1)
            inside = {a for a in addrs if pl <= 32 and (pl == 0 or (a ^ net) >> (32 - pl) == 0)}
            r["addrs_outside"] = len(addrs) - len(inside)
        else:
            r["addrs_outside"] = len(addrs)
        r["prefix_hosts"] = hosts
        r["permille"] = (int(r["addrs"]) - int(r["addrs_outside"])) * 1000 // hosts if hosts else 0
        for m in range(3):
            ips = [e[2] for e in live if e[0] == m]
            r["conflicts"] += sum(1 for a in set(ips) if ips.count(a) > 1)
    macs = set(np.ascontiguousarray(d["subscriber_pools"][0]).view("<u8").reshape(-1).tolist())
    cid_vals = np.ascontiguousarray(d["circuit_id_map"][1]).view("<u8").reshape(-1).tolist()
    summary = {
        "entries": [sum(1 for e in ent if e[0] == m and not e[3]) for m in range(3)],
        "expired": [sum(1 for e in ent if e[0] == m and e[3]) for m in range(3)],
        "addrs": len({e[2] for e in ent if not e[3]}),
        "conflicts": int(recs["conflicts"].sum()),
        "unknown_pool": sum(1 for e in ent if not e[3] and e[1] not in pools),
        "cid_dangling": sum(1 for v in cid_vals if v not in macs),
        "pools_found": len(ids),
    }
    return summary, np.array(ids, "<u4"), recs


def _pa_pool(v):
    return np.ascontiguousarray(v).view(L.ip_pool).reshape(-1) if len(v) else np.zeros(0, L.ip_pool)


def due_rule(d, now_ns, grace_s=0):
    """The sweep's due set as bng_lease_removed records sorted as Dataplane.lease_sweep sorts them, and the
    circuit_id_map keys that go with it."""
    now_s = now_ns // NS
    rows = []
    for m, name in enumerate(LEASE_MAPS):
        k, v = d[name]
        a = _pa(v)
        for i in range(len(a)):
            if now_s > min(int(a["lease_expiry"][i]) + grace_s, U64_MAX):
                r = np.zeros(1, L.bng_lease_removed)[0]
                r["key"][:k.shape[1]] = k[i]
                for f in ("lease_expiry", "pool_id", "allocated_ip", "vlan_id", "client_class", "flags"):
                    r[f] = a[f][i]
                r["map"] = m
                rows.append(r)
    out = np.array(rows, L.bng_lease_removed) if rows else np.zeros(0, L.bng_lease_removed)
    o = np.lexsort([out["key"][:, j] for j in range(31, -1, -1)] + [out["map"]])
    return out[o]


def minus(d, removed):
    """The five dumps without the removed records and the circuit_id_map entries of the removed MACs."""
    out = dict(d)
    gone_macs = set()
    for m, name in enumerate(LEASE_MAPS):
        k, v = d[name]
        gone = {bytes(r["key"][:k.shape[1]]) for r in removed if r["map"] == m}
        keep = np.array([bytes(x) not in gone for x in k], bool) if len(k) else np.zeros(0, bool)
        out[name] = (k[keep], v[keep])
        if m == 0:
            gone_macs = {int.from_bytes(g, "little") for g in gone}
    k, v = d["circuit_id_map"]
    vals = np.ascontiguousarray(v).view("<u8").reshape(-1).tolist()
    keep = np.array([x not in gone_macs for x in vals], bool) if len(k) else np.zeros(0, bool)
    out["circuit_id_map"] = (k[keep], v[keep])
    return out


def same_dumps(a, b, what):
    for m in DHCP_MAPS:
        assert a[m][0].tobytes() == b[m][0].tobytes() and a[m][1].tobytes() == b[m][1].tobytes(), f"{what}: {m} differs"


def check_census(dp, now_ns, what, wire=True):
    dp.lease_addr_order(wire)
    d = _dumps(dp)
    ws, wi, wr = census_rule(d, now_ns, wire)
    gs, gi, gr = dp.lease_census(now_ns)
    assert gs == ws, f"{what}: summary {gs} != {ws}"
    assert gi.tolist() == wi.tolist(), f"{what}: pool ids"
    for f in POOL_FIELDS:
        assert np.array_equal(gr[f], wr[f]), f"{what}: {f}: {gr[f].tolist()} != {wr[f].tolist()}"
    assert not gr["pad"].any()
    assert dp.lease_census(now_ns)[2].tobytes() == gr.tobytes(), f"{what}: a second census differs"
    for cap in (0, 1, max(len(wi) - 1, 0), len(wi) + 5):
        cs, ci, cr = dp.lease_census(now_ns, cap=cap)
        assert cs == ws and len(ci) == min(cap, len(wi)), f"{what}: cap {cap}"
        pos = np.searchsorted(wi, ci)
        assert np.array_equal(wi[pos], ci) and cr.tobytes() == gr[pos].tobytes(), f"{what}: cap {cap} records"
    return gs


# ---------------------------------------------------------------------------
# tables
# ---------------------------------------------------------------------------
def load_dhcp_script(be):
    """The map updates of the `dhcp` golden script; returns the script."""
    sc = scenarios.ALL_SCRIPTS["dhcp"]()
    for st in sc.steps:
        if st[0] == "update":
            assert be.update(st[1], st[2], st[3], st[4]) == 0
    return sc


def cid_key(b: bytes):
    k = np.zeros(32, np.uint8)
    k[:len(b)] = np.frombuffer(b, np.uint8)
    return k


def constructed(now_s=NOW_S):
    """Updates [(map, keys, values)] built for the census and the sweep: see the comments."""
    n = 40
    macs = S.sub_mac_key(np.arange(n))
    pa = np.zeros(n, L.pool_assignment)
    pa["pool_id"] = 1 + np.arange(n) % 6                     # pools 1-4 exist (prefix 24, 0, 32, 33); 5 and 6 do not
    pa["allocated_ip"] = S.ip_bytes(np.uint32(0x0A000100) + np.arange(n))
    pa["lease_expiry"] = now_s + (np.arange(n) % 3) - 1      # now_s - 1 (expired), now_s, now_s + 1: strict >
    pa["vlan_id"], pa["client_class"], pa["flags"] = np.arange(n), np.arange(n) % 7, np.arange(n) % 3
    pa["lease_expiry"][30] = U64_MAX                         # the grace sum saturates
    pa["allocated_ip"][7] = pa["allocated_ip"][1]            # the same address under two MACs of pool 2: a conflict (and one more in the VLAN map below)
    pa["lease_expiry"][1] = pa["lease_expiry"][7] = now_s + 5
    pa["allocated_ip"][13] = pa["allocated_ip"][19]          # two MACs of pool 2, one of them expired: no conflict
    pa["lease_expiry"][13], pa["lease_expiry"][19] = now_s - 1, now_s + 5
    pa["allocated_ip"][6] = [192, 168, 0, 1]                 # pool 1 (10.0.1.0/24): outside its prefix
    pa["lease_expiry"][6] = now_s + 5
    pools = np.zeros(4, L.ip_pool)
    pools["network"] = [[10, 0, 1, 0], [0, 0, 0, 0], [10, 0, 1, 2], [10, 0, 1, 0]]
    pools["prefix_len"] = [24, 0, 32, 33]
    pools["gateway"] = [[10, 0, 1, 1]] * 4
    pools["lease_time"] = 3600
    vk = np.zeros(8, L.vlan_key)
    vk["s_tag"], vk["c_tag"] = 100 + np.arange(8), [0, 0, 0, 0, 7, 7, 7, 7]
    vpa = pa[:8].copy()                                      # subscribers 0-7 also by VLAN, same addresses: no conflict
    vpa["lease_expiry"][0] = now_s - 10                      # ... but subscriber 0's VLAN entry has expired
    ck = np.stack([cid_key(b"port %d" % i) for i in range(4, 12)])
    cpa = pa[4:12].copy()                                    # subscribers 4-11 also by circuit-id
    cpa["allocated_ip"][7] = cpa["allocated_ip"][6]          # two circuit-ids of pool 5 with one address: a conflict
    cpa["pool_id"][7] = cpa["pool_id"][6]
    cpa["lease_expiry"][6:8] = now_s + 9
    cm_k = np.arange(1, 9, dtype="<u8") * np.uint64(0x9E3779B97F4A7C15)
    cm_v = macs[[0, 1, 2, 13, 28, 29, 30, 31]].copy()
    cm_v[7] = np.uint64(0x02FFFFFFFFFF)                      # dangling: no such subscriber
    return [("ip_pools", np.arange(1, 5, dtype="<u4"), pools), ("subscriber_pools", macs, pa), ("vlan_subscriber_pools", vk, vpa),
            ("circuit_id_subscribers", ck, cpa), ("circuit_id_map", cm_k, cm_v)]


def load(be, ups):
    for m, k, v in ups:
        assert be.update(m, as_bytes(k), as_bytes(v), 0) == 0, m


# ---------------------------------------------------------------------------
# census
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("now_s", [0, 3, 4, NOW_S])
def test_census_on_the_dhcp_script(now_s):
    be = harness.GpuBackend()
    try:
        harness.run_script(be, scenarios.ALL_SCRIPTS["dhcp"]())
        s = check_census(be.dp, now_s * NS + 999_999_999, f"dhcp script at {now_s}")
        assert sum(s["entries"]) + sum(s["expired"]) > 60 and (s["unknown_pool"] > 0 or now_s >= 4)
    finally:
        be.close()


@pytest.mark.parametrize("dt", [-2, -1, 0, 1, 2, 6, 10])
def test_census_on_constructed_tables(dt):
    with _small() as dp:
        load(harness.GpuBackend(dp), constructed())
        # the same bytes read as numeric words: only addrs_outside and permille may differ, and the rule says how
        n = check_census(dp, (NOW_S + dt) * NS + 5, f"constructed at {dt:+d}, numeric order", wire=False)
        s = check_census(dp, (NOW_S + dt) * NS + 5, f"constructed at {dt:+d}")
        assert n == s
        assert s["cid_dangling"] == 1
        if dt == 0:
            assert s["conflicts"] == 3 and s["expired"][0] > 0 and s["unknown_pool"] > 0
            ids, recs = dp.lease_census(NOW_S * NS)[1:]
            by = {int(i): r for i, r in zip(ids, recs)}
            dp.lease_addr_order(False)
            assert dp.lease_census(NOW_S * NS)[2]["addrs_outside"].tolist() != recs["addrs_outside"].tolist()
            assert by[1]["addrs_outside"] == 1 and by[2]["conflicts"] == 2 and by[5]["conflicts"] == 1
            assert by[4]["prefix_hosts"] == 0 and by[4]["addrs_outside"] == by[4]["addrs"] and by[2]["prefix_hosts"] == 2**32 - 1
            assert not by[5]["known"] and by[3]["prefix_hosts"] == 1


def test_census_with_many_unknown_pools():
    """More pool ids without an ip_pools entry than the scratch hash starts with: it grows and the census runs again."""
    n = 20_000
    with _small(max_subscribers=1 << 15) as dp:
        pa = np.zeros(n, L.pool_assignment)
        pa["pool_id"] = 100 + np.arange(n)
        pa["allocated_ip"] = S.ip_bytes(np.uint32(0x0A000000) + np.arange(n) // 2)
        pa["lease_expiry"] = 10
        assert dp.update_batch("subscriber_pools", as_bytes(S.sub_mac_key(np.arange(n))), as_bytes(pa)) == 0
        s, ids, recs = dp.lease_census(5 * NS)
        assert s["pools_found"] == n and s["unknown_pool"] == n and s["addrs"] == n // 2 and s["conflicts"] == 0
        assert ids.tolist() == list(range(100, 100 + n)) and (recs["addrs"] == 1).all() and (recs["addrs_outside"] == 1).all()
        assert dp.lease_census(11 * NS)[0]["expired"] == [n, 0, 0]


def test_one_unknown_pool_with_many_leases_is_one_pass():
    """Threads racing to give one unknown pool_id its record claim one slot between them: the hash does not overflow and
    the census is its two kernels, once."""
    n = 200_000
    with _small(max_subscribers=1 << 18) as dp:
        pa = np.zeros(n, L.pool_assignment)
        pa["pool_id"], pa["lease_expiry"] = 77, 10
        pa["allocated_ip"] = S.ip_bytes(np.uint32(0x0A000000) + np.arange(n))
        assert dp.update_batch("subscriber_pools", as_bytes(S.sub_mac_key(np.arange(n))), as_bytes(pa)) == 0
        for _ in range(3):
            l0 = dp.launch_count
            s, ids, recs = dp.lease_census(5 * NS, cap=4)
            assert dp.launch_count - l0 == 2
            assert ids.tolist() == [77] and recs["entries"][0].tolist() == [n, 0, 0] and s["unknown_pool"] == n


def _frames(fs):
    lens = np.array([len(f) for f in fs], np.uint32)
    width = int(((lens.max() + 15) // 16) * 16)
    arena = np.zeros((len(fs), width), np.uint8)
    for i, f in enumerate(fs):
        arena[i, :len(f)] = f
    return arena.reshape(-1), lens, width


def _opt82(cid: bytes, rid=b"rid"):
    sub = bytes([1, len(cid)]) + cid + bytes([2, len(rid)]) + rid
    return bytes([82, len(sub)]) + sub


@pytest.mark.parametrize("dt", [-1, 0, 1, 6, 10])
def test_census_agrees_with_the_program(dt):
    """cache_expired grows by the frames whose first-found entry (VLAN pair, then circuit-id, then chaddr) is expired by
    the census's rule, with the entries looked up in the dumps."""
    ups = constructed()
    now_ns = (NOW_S + dt) * NS + 7
    unknown = 0x02DEAD000001
    # (frame, the keys the program tries: VLAN pair, circuit-id, MAC word; None: the frame does not carry it)
    probes = []
    for m in ups[1][1]:
        probes.append((scenarios.dhcp_frame(int(m), msg_type=3), None, None, int(m)))
    for k in ups[2][1]:
        if k["c_tag"] == 0:  # by VLAN pair first, whatever the MAC
            probes.append((scenarios.dhcp_frame(int(ups[1][1][3]), vlan=((0x8100, int(k["s_tag"])),), frame_len=380),
                           bytes(as_bytes(k[None])[0]), None, int(ups[1][1][3])))
    for i in range(2, 14):  # by circuit-id before the MAC; "port 2", "port 3", "port 12", "port 13" have no entry
        cid = b"port %d" % i
        probes.append((scenarios.dhcp_frame(int(ups[1][1][20]), extra_opts=_opt82(cid)), None, bytes(cid_key(cid)), int(ups[1][1][20])))
        probes.append((scenarios.dhcp_frame(unknown, extra_opts=_opt82(cid)), None, bytes(cid_key(cid)), unknown))
    with _small() as dp:
        load(harness.GpuBackend(dp), ups)
        d = _dumps(dp)
        exp = [{bytes(k): int(e) for k, e in zip(d[m][0], _pa(d[m][1])["lease_expiry"])} for m in LEASE_MAPS]
        want = cid_first = 0
        for _, vk, ck, mac in probes:
            first = None
            if vk is not None:
                first = exp[1].get(vk)
            if first is None and ck is not None:
                first = exp[2].get(ck)
                cid_first += first is not None
            if first is None:
                first = exp[0].get(int(mac).to_bytes(8, "little"))
            want += first is not None and now_ns // NS > first
        assert cid_first == 16
        before = dp.stats("stats_map")[4]
        arena, lens, width = _frames([p[0] for p in probes])
        dp.run("dhcp_fastpath_prog", arena, lens, now_ns, stride=width)
        assert int(dp.stats("stats_map")[4] - before) == want and (want > 0 or dt < 0)
        s = census_rule(d, now_ns)[0]
        assert dp.lease_census(now_ns)[0]["expired"] == s["expired"]


def test_census_is_pure():
    """Dumps, stats_map, events, launch counts of program runs and a delta export: the same with and without censuses."""
    def session(census):
        be = harness.GpuBackend()
        dp = be.dp
        try:
            dp.delta_enable()
            sc = load_dhcp_script(be)
            run = [st for st in sc.steps if st[0] == "run"][0]
            first = dp.delta_export(full=True)
            launches = []
            for rep in range(3):
                if census:
                    dp.lease_census((rep + 2) * NS)
                a, l = run[2].copy(), run[3].copy()
                l0 = dp.launch_count
                v = dp.run(run[1], a, l, run[4], off16=run[5], stride=run[6])
                launches.append(dp.launch_count - l0)
                if census:
                    dp.lease_census(NOW_S * NS, cap=2)
            dp.delta_export(exact=True)
            before = dp.delta_info()
            if census:
                dp.lease_census(4 * NS)
            nothing = dp.delta_export(exact=True)
            return (_dumps(dp), dp.stats("stats_map").tobytes(), [dp.drain(m).tobytes() for m in harness.EVENT_MAPS], launches,
                    v.tobytes(), a.tobytes(), len(first), len(nothing), dp.delta_info()[1] - before[1])
        finally:
            be.close()

    a, b = session(False), session(True)
    same_dumps(a[0], b[0], "census purity")
    assert a[1:] == b[1:]


# ---------------------------------------------------------------------------
# sweep
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("dt,grace", [(-2, 0), (0, 0), (1, 0), (1, 1), (2, 1), (6, 0), (10, 3), (10, 2**32 - 1)])
def test_sweep_against_the_rule(dt, grace):
    now_ns = (NOW_S + dt) * NS + 3
    with _small() as dp:
        load(harness.GpuBackend(dp), constructed())
        d0 = _dumps(dp)
        want = due_rule(d0, now_ns, grace)
        info0 = {m: dp.map_info(m) for m in DHCP_MAPS}
        stats0 = dp.stats("stats_map").tobytes()
        found, none, removed = dp.lease_sweep(now_ns, grace, cap=0)  # the dry run
        assert found == len(want) and len(none) == 0 and removed == [0, 0, 0, 0]
        same_dumps(_dumps(dp), d0, "dry run")
        found, got, removed = dp.lease_sweep(now_ns, grace)
        assert found == len(want) and got.tobytes() == want.tobytes()
        d1 = _dumps(dp)
        exp = minus(d0, want)
        same_dumps(d1, exp, "after the sweep")
        assert removed[:3] == [int((want["map"] == m).sum()) for m in range(3)]
        assert removed[3] == len(d0["circuit_id_map"][0]) - len(exp["circuit_id_map"][0])
        for m in DHCP_MAPS:
            assert dp.map_info(m)["count"] == len(exp[m][0]) and dp.map_info(m)["max_entries"] == info0[m]["max_entries"]
            assert info0[m]["count"] - dp.map_info(m)["count"] == len(d0[m][0]) - len(exp[m][0])
        assert dp.stats("stats_map").tobytes() == stats0
        assert dp.lease_sweep(now_ns, grace)[0] == 0, "a second sweep finds nothing"
        same_dumps(_dumps(dp), d1, "second sweep")
        check_census(dp, now_ns, "census after the sweep")
        if grace == 0:
            assert dp.lease_census(now_ns)[0]["expired"] == [0, 0, 0]


@pytest.mark.parametrize("cap", [1, 3, 7])
def test_capped_sweeps_converge(cap):
    now_ns = (NOW_S + 20) * NS
    with _small() as one, _small() as dp:
        load(harness.GpuBackend(one), constructed())
        load(harness.GpuBackend(dp), constructed())
        one.lease_sweep(now_ns)
        final = _dumps(one)
        seen = []
        while True:
            d0 = _dumps(dp)
            found, got, removed = dp.lease_sweep(now_ns, cap=cap)
            assert len(got) == min(found, cap) and sum(removed[:3]) == len(got)
            same_dumps(_dumps(dp), minus(d0, got), f"cap {cap}: exactly the reported entries went")
            seen += [(int(r["map"]), bytes(r["key"])) for r in got]
            if found <= cap:
                break
        assert len(seen) == len(set(seen)) == len(due_rule(_dumps_of(constructed()), now_ns))
        same_dumps(_dumps(dp), final, f"cap {cap}: converged")


def _dumps_of(ups):
    with _small() as dp:
        load(harness.GpuBackend(dp), ups)
        return _dumps(dp)


def _oracle_kind():
    return "reference" if pyoracle.available("reference") else "port"


def _replay_after(ups, now_ns, steps, sweep_now):
    """GPU: load, sweep at sweep_now, run `steps`; oracle: load, delete the swept keys by map commands, run them.
    Returns both results of harness.run_script for the steps."""
    sc = harness.Script("after sweep")
    sc.steps = list(steps)
    be = harness.GpuBackend()
    try:
        load(be, ups)
        d0 = _dumps(be.dp)
        found, removed, _ = be.dp.lease_sweep(sweep_now)
        gone = minus(d0, removed)
        got = harness.run_script(be, sc)
    finally:
        be.close()
    ob = harness.OracleBackend(_oracle_kind())
    try:
        load(ob, ups)
        for m in LEASE_MAPS + ("circuit_id_map",):
            kept = {bytes(k) for k in gone[m][0]}
            for k in d0[m][0]:
                if bytes(k) not in kept:
                    assert ob.delete(m, k) == 0
        want = harness.run_script(ob, sc)
    finally:
        ob.close()
    return want, got, removed


def test_expired_vlan_entry_no_longer_shadows_the_fresh_lease():
    ups = constructed()
    ups[2][2]["lease_expiry"][1] = NOW_S - 10  # subscriber 1: a fresh lease by MAC in a known pool, an expired VLAN entry
    now_ns = NOW_S * NS
    f = scenarios.dhcp_frame(int(S.sub_mac_key(1)), msg_type=3, vlan=((0x8100, 101),), frame_len=380)
    arena, lens, width = _frames([f])
    with _small() as dp:
        load(harness.GpuBackend(dp), ups)
        assert dp.run("dhcp_fastpath_prog", arena.copy(), lens.copy(), now_ns, stride=width).tolist() == [2]  # XDP_PASS
    want, got, removed = _replay_after(ups, now_ns, [("run", "dhcp_fastpath_prog", arena, lens, now_ns, None, width, None, None)], now_ns)
    assert any(r["map"] == 1 and bytes(r["key"][:4]) == bytes([101, 0, 0, 0]) for r in removed)
    harness.compare(want, got, "reply after the sweep")
    assert got["s000_verdict"].tolist() == [3]  # XDP_TX


@pytest.mark.parametrize("sweep_s", [4, NOW_S])
def test_dhcp_script_continues_bit_exact_after_a_sweep(sweep_s):
    sc = scenarios.ALL_SCRIPTS["dhcp"]()
    ups = [(st[1], st[2], st[3]) for st in sc.steps if st[0] == "update"]
    rest = [st for st in sc.steps if st[0] != "update"]
    want, got, removed = _replay_after(ups, 0, rest, sweep_s * NS)
    assert len(removed) > 0
    harness.compare(want, got, f"dhcp script after a sweep at {sweep_s}")


def test_capacity_and_rebuild():
    from bng_b200 import Dataplane
    n = 512
    with Dataplane(max_batch=1 << 10, max_subscribers=n, max_nat_sessions=1 << 10, max_eim_mappings=1 << 10) as dp:
        assert dp.map_info("subscriber_pools")["max_entries"] == n
        pa = np.zeros(n, L.pool_assignment)
        pa["pool_id"], pa["lease_expiry"] = 1, 10
        pa["allocated_ip"] = S.ip_bytes(np.uint32(0x0A000000) + np.arange(n))
        assert dp.update_batch("subscriber_pools", as_bytes(S.sub_mac_key(np.arange(n))), as_bytes(pa)) == 0
        assert dp.update("subscriber_pools", np.uint64(0x02AA00000000), pa[:1]) != 0, "the table is full"
        cm = np.arange(1, n + 1, dtype="<u8")
        assert dp.update_batch("circuit_id_map", as_bytes(cm), as_bytes(S.sub_mac_key(np.arange(n)))) == 0
        flow0, lease0 = dp.table_rebuilds, dp.lease_table_rebuilds()
        found, got, removed = dp.lease_sweep(11 * NS)
        assert found == n and removed == [n, 0, 0, n]
        assert dp.lease_table_rebuilds() == lease0 + 2 and dp.table_rebuilds == flow0
        assert dp.map_info("subscriber_pools")["count"] == 0 and dp.map_info("circuit_id_map")["count"] == 0
        pa["lease_expiry"] = 1 << 40
        for i in range(n):  # one by one: every insert must find room
            assert dp.update("subscriber_pools", np.uint64(0x02BB00000000 + i), pa[i:i + 1]) == 0, i
        assert dp.map_info("subscriber_pools")["count"] == n
        assert dp.lease_census(12 * NS)[0]["entries"] == [n, 0, 0]


@pytest.mark.parametrize("mass", [False, True])
def test_replication_carries_the_removals(mass):
    """mass: enough entries go for the tables to be rebuilt before the export."""
    from bng_b200 import Dataplane
    opts = dict(max_batch=1 << 10, max_subscribers=256, max_nat_sessions=1 << 10, max_eim_mappings=1 << 10)
    with Dataplane(**opts) as act, Dataplane(**opts) as sby:
        load(harness.GpuBackend(act), constructed())
        if mass:
            n = 200
            pa = np.zeros(n, L.pool_assignment)
            pa["pool_id"], pa["lease_expiry"] = 2, NOW_S - 5 + np.arange(n) % 10
            pa["allocated_ip"] = S.ip_bytes(np.uint32(0x0B000000) + np.arange(n))
            assert act.update_batch("subscriber_pools", as_bytes(S.sub_mac_key(1000 + np.arange(n))), as_bytes(pa)) == 0
        act.delta_enable()
        assert sby.delta_apply(act.delta_export(full=True)) == 0
        same_dumps(_dumps(sby), _dumps(act), "standby after the full delta")
        r0 = act.lease_table_rebuilds()
        found = act.lease_sweep((NOW_S + 2) * NS)[0]
        assert found > 0 and (act.lease_table_rebuilds() > r0) == mass
        assert sby.delta_apply(act.delta_export()) == 0
        same_dumps(_dumps(sby), _dumps(act), "standby after the sweep's delta")
        assert sby.lease_census(NOW_S * NS)[2].tobytes() == act.lease_census(NOW_S * NS)[2].tobytes()


def test_error_codes():
    with _small() as dp:
        lib, h = dp.lib, dp.h
        s = np.zeros(1, L.bng_lease_sum)
        ids, out = np.zeros(4, "<u4"), np.zeros(4, L.bng_lease_pool_use)
        rem = np.zeros(4, L.bng_lease_removed)
        assert lib.bng_dhcp_lease_census(h, 0, s.ctypes.data, ids.ctypes.data, out.ctypes.data, 4) == 0
        assert lib.bng_dhcp_lease_census(None, 0, s.ctypes.data, ids.ctypes.data, out.ctypes.data, 4) == -errno.EINVAL
        assert lib.bng_dhcp_lease_census(h, 0, None, ids.ctypes.data, out.ctypes.data, 4) == -errno.EINVAL
        assert lib.bng_dhcp_lease_census(h, 0, s.ctypes.data, None, out.ctypes.data, 1) == -errno.EINVAL
        assert lib.bng_dhcp_lease_census(h, 0, s.ctypes.data, ids.ctypes.data, None, 1) == -errno.EINVAL
        assert lib.bng_dhcp_lease_census(h, 0, s.ctypes.data, None, None, 0) == 0
        assert lib.bng_dhcp_lease_sweep(None, 0, 0, rem.ctypes.data, 4, None) == -errno.EINVAL
        assert lib.bng_dhcp_lease_sweep(h, 0, 0, None, 1, None) == -errno.EINVAL
        assert lib.bng_dhcp_lease_sweep(h, 0, 0, None, 0, None) == 0
        assert lib.bng_dhcp_lease_sweep(h, 0, 0, rem.ctypes.data, 2**40, None) == 0
        assert lib.bng_lease_table_rebuilds(None) == 0
