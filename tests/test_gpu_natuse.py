"""NAT port-usage census (bng_nat_usage): the GPU's records against the definitions of include/bng_b200.h, restated
here in numpy (nat_usage_rule) over the dumps of subscriber_nat, nat_sessions, eim_table and nat_reverse.

The definitions, restated:
  - a live session holds (nat_ip, ntohs(nat_port), protocol); a live EIM entry holds (external_ip, external_port,
    key.protocol), external_port in host order;
  - a session is attributed to its key src_ip, an EIM entry to its key internal_ip;
  - protocol columns [0] TCP, [1] UDP, [2] ICMP; other protocol bytes count in the totals and *_any only;
  - a session is unreachable when nat_reverse has no entry under (dst_ip, nat_ip, dst_port, nat_port, protocol, 0),
    or one whose value is not the session's key; a reverse entry is stale when its value keys no live session;
  - per subscriber_nat entry with block B = (public_ip, [port_start, port_end]): the distinct ports of B it holds per
    column and with any protocol, the distinct triples it holds outside B, its sessions, EIM entries and unreachable
    sessions, and permille = floor(max(in_use) * 1000 / block_ports);
  - per public address (a block's public_ip or a held triple's): entries holding a triple on it, the blocks on it and
    their ports, the distinct ports held on it per column and with any protocol, its unreachable sessions."""
import errno

import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import layouts as L
from bng_b200 import synth as S
from bng_b200 import workloads as W
from bng_b200.layouts import as_bytes
from test_gpu_acct import FEED_IDS, FEEDS, _pipeline_batch
from test_oracle_fuzz import fuzz_script

pytestmark = pytest.mark.gpu

NAT_MAPS = ("subscriber_nat", "nat_sessions", "eim_table", "nat_reverse")
SCRIPTS = [s for s in sorted(scenarios.ALL_SCRIPTS) if s.startswith(("nat", "pipeline")) or s in ("ticks", "ipopts")]
SUB_FIELDS = [f for f in L.bng_nat_sub_use.names if f != "pad"]
PUB_FIELDS = [f for f in L.bng_nat_pub_use.names if f != "pad"]


# ---------------------------------------------------------------------------
# the rule, restated
# ---------------------------------------------------------------------------
def _u4(b):
    return np.ascontiguousarray(b).view("<u4").reshape(-1) if len(b) else np.zeros(0, np.uint32)


def _w2(b16):
    """16-byte keys -> (n, 2) u64 words."""
    return np.ascontiguousarray(b16).view("<u8").reshape(-1, 2) if len(b16) else np.zeros((0, 2), np.uint64)


def _find(table, queries):
    """Index in `table` (unique (n, 2) u64 rows) of every query row, or -1."""
    n, m = len(table), len(queries)
    if m == 0:
        return np.zeros(0, np.int64)
    if n == 0:
        return np.full(m, -1, np.int64)
    allk = np.concatenate([table, queries])
    tag = np.concatenate([np.zeros(n, np.int64), np.ones(m, np.int64)])
    order = np.lexsort((tag, allk[:, 1], allk[:, 0]))
    pos = np.where(tag[order] == 0, np.arange(n + m), -1)
    last = np.maximum.accumulate(pos)  # the last table row at or before each sorted position
    res = np.full(n + m, -1, np.int64)
    ok = last >= 0
    cand = np.where(ok, order[np.maximum(last, 0)], 0)
    ok &= (allk[cand] == allk[order]).all(axis=1)
    res[order] = np.where(ok, cand, -1)
    return res[n:]


def _count_by(keys, uniq_keys):
    """How often each of uniq_keys occurs in keys."""
    if len(uniq_keys) == 0:
        return np.zeros(0, np.int64)
    u, c = np.unique(keys, return_counts=True)
    idx = np.searchsorted(u, uniq_keys)
    idx = np.minimum(idx, max(len(u) - 1, 0))
    return np.where((len(u) > 0) & (u[idx] == uniq_keys) if len(u) else False, c[idx] if len(u) else 0, 0)


def _col(proto):
    return np.select([proto == 6, proto == 17, proto == 1], [0, 1, 2], -1)


def nat_usage_rule(dumps, min_permille=0):
    """dumps: {map: (keys u8[n, ks], values u8[n, vs])} of NAT_MAPS.  Returns (summary dict, subscriber addresses,
    sub records, public addresses, pub records), each kind sorted by address bytes, as Dataplane.nat_usage returns."""
    nk, nv = dumps["subscriber_nat"]
    sk, sv = dumps["nat_sessions"]
    ek, ev = dumps["eim_table"]
    rk, rv = dumps["nat_reverse"]
    sub_addr = _u4(nk[:, :4])
    b_ip = _u4(nv[:, 0:4])
    b_ps = nv[:, 4].astype(np.int64) | nv[:, 5].astype(np.int64) << 8
    b_pe = nv[:, 6].astype(np.int64) | nv[:, 7].astype(np.int64) << 8
    b_ports = np.where(b_pe >= b_ps, b_pe - b_ps + 1, 0)

    # held triples
    s_proto = sv[:, 73].astype(np.int64) if len(sv) else np.zeros(0, np.int64)
    s_ip = _u4(sv[:, 0:4]).astype(np.int64)
    s_port = (sv[:, 4].astype(np.int64) << 8 | sv[:, 5].astype(np.int64)) if len(sv) else np.zeros(0, np.int64)
    s_attr = _u4(sk[:, 0:4]).astype(np.int64)
    rev_q = np.zeros((len(sk), 16), np.uint8)
    if len(sk):
        rev_q[:, 0:4], rev_q[:, 4:8], rev_q[:, 8:10], rev_q[:, 10:12] = sk[:, 4:8], sv[:, 0:4], sk[:, 10:12], sv[:, 4:6]
        rev_q[:, 12] = sv[:, 73]
    ri = _find(_w2(rk), _w2(rev_q))
    unr = ri < 0
    if len(sk):
        hit = ~unr
        unr[hit] = ~(_w2(rv)[ri[hit]] == _w2(sk)[hit]).all(axis=1)
    stale = int((_find(_w2(sk), _w2(rv)) < 0).sum())

    e_ip = _u4(ev[:, 0:4]).astype(np.int64)
    e_port = (ev[:, 4].astype(np.int64) | ev[:, 5].astype(np.int64) << 8) if len(ev) else np.zeros(0, np.int64)
    e_proto = ek[:, 6].astype(np.int64) if len(ek) else np.zeros(0, np.int64)
    e_attr = _u4(ek[:, 0:4]).astype(np.int64)

    ip = np.concatenate([s_ip, e_ip])
    port = np.concatenate([s_port, e_port])
    proto = np.concatenate([s_proto, e_proto])
    attr = np.concatenate([s_attr, e_attr])
    is_ses = np.concatenate([np.ones(len(s_ip), bool), np.zeros(len(e_ip), bool)])
    h_unr = np.concatenate([unr, np.zeros(len(e_ip), bool)])
    trip = ip | port << 32 | proto << 48
    col = _col(proto)

    # per public address
    pubs = np.unique(np.concatenate([b_ip.astype(np.int64), ip]))
    ut, ut_i = np.unique(trip, return_index=True)
    pairs = np.unique(ip | port << 32)
    pub = np.zeros(len(pubs), L.bng_nat_pub_use)
    pub["sessions"] = _count_by(ip[is_ses], pubs)
    pub["eim"] = _count_by(ip[~is_ses], pubs)
    pub["blocks"] = _count_by(b_ip.astype(np.int64), pubs)
    pi = np.searchsorted(pubs, b_ip.astype(np.int64))
    bp = np.zeros(len(pubs), np.int64)
    np.add.at(bp, pi, b_ports)
    pub["block_ports"] = bp
    for c in range(3):
        pub["in_use"][:, c] = _count_by(ut[_col(ut >> 48) == c] & 0xFFFFFFFF, pubs)
    pub["in_use_any"] = _count_by(pairs & 0xFFFFFFFF, pubs)
    pub["unreachable"] = _count_by(ip[h_unr], pubs)

    # per subscriber
    order = np.argsort(sub_addr)
    sa_sorted = sub_addr[order].astype(np.int64)
    j = np.searchsorted(sa_sorted, attr)
    j = np.minimum(j, max(len(sa_sorted) - 1, 0))
    owned = (sa_sorted[j] == attr) if len(sa_sorted) else np.zeros(len(attr), bool)
    row = np.where(owned, order[j] if len(order) else 0, -1)
    sub = np.zeros(len(sub_addr), L.bng_nat_sub_use)
    sub["public_ip"], sub["block_ports"] = b_ip, b_ports
    o = owned
    r_, ip_, port_, col_, tr_ = row[o], ip[o], port[o], col[o], trip[o]
    inside = (ip_ == b_ip[r_].astype(np.int64)) & (port_ >= b_ps[r_]) & (port_ <= b_pe[r_])
    ar = np.arange(len(sub_addr))
    sub["sessions"] = _count_by(r_[is_ses[o]], ar)
    sub["eim"] = _count_by(r_[~is_ses[o]], ar)
    sub["unreachable"] = _count_by(r_[h_unr[o]], ar)
    for c in range(3):
        m = inside & (col_ == c)
        sub["in_use"][:, c] = _count_by(np.unique(r_[m] << 16 | port_[m]) >> 16, ar)
    sub["in_use_any"] = _count_by(np.unique(r_[inside] << 16 | port_[inside]) >> 16, ar)
    out_rows = np.unique(np.stack([r_[~inside], tr_[~inside]], axis=1), axis=0) if (~inside).any() else np.zeros((0, 2), np.int64)
    sub["outside"] = _count_by(out_rows[:, 0], ar)
    mx = sub["in_use"].max(axis=1).astype(np.int64) if len(sub) else np.zeros(0, np.int64)
    sub["permille"] = np.where(b_ports > 0, mx * 1000 // np.maximum(b_ports, 1), 0)

    summary = {
        "subscribers": len(sub_addr), "sessions": len(sk), "eim": len(ek), "triples": len(ut),
        "unreachable": int(unr.sum()), "stale_reverse": stale,
        "orphan_sessions": int((~owned[is_ses]).sum()), "orphan_eim": int((~owned[~is_ses]).sum()),
    }
    q = sub["permille"] >= min_permille
    sa, sub = sub_addr[q], sub[q]
    summary["subs_found"], summary["pubs_found"] = len(sa), len(pubs)
    pa = pubs.astype(np.uint32)
    os_, op = np.argsort(sa.byteswap(), kind="stable"), np.argsort(pa.byteswap(), kind="stable")
    return summary, sa[os_], sub[os_], pa[op], pub[op]


def _dumps(be):
    return {m: be.dump(m) for m in NAT_MAPS}


def check_census(dp, dumps, what, min_permille=0):
    """dp's census equals the rule over `dumps`, field by field; returns the rule's result."""
    got = dp.nat_usage(min_permille)
    want = nat_usage_rule(dumps, min_permille)
    assert got[0] == want[0], f"{what}: summary {got[0]} vs rule {want[0]}"
    assert np.array_equal(got[1], want[1]), f"{what}: subscriber addresses differ"
    assert np.array_equal(got[3], want[3]), f"{what}: public addresses differ"
    for f in SUB_FIELDS:
        assert np.array_equal(got[2][f], want[2][f]), f"{what}: subscriber field {f} differs"
    for f in PUB_FIELDS:
        assert np.array_equal(got[4][f], want[4][f]), f"{what}: public-address field {f} differs"
    assert not got[2]["pad"].any() and not got[4]["pad"].any(), f"{what}: padding not zero"
    return want


def run_census(script_fn, pinned, ora_kind, **opts):
    """Runs the script on the GPU step by step beside the oracle; after every step the verdicts and frames equal the
    oracle's and the census equals the rule over the oracle's tables.  Returns the rule's last result."""
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    want = harness.run_script(harness.OracleBackend(ora_kind), script_fn())
    script = script_fn()
    be = harness.GpuBackend(pinned=pinned, **opts)
    rep = harness.OracleBackend(ora_kind)
    last = None
    try:
        for si, st in enumerate(script.steps):
            tag = f"s{si:03d}"
            if st[0] == "update":
                be.update(st[1], st[2], st[3], st[4])
                rep.update(st[1], st[2], st[3], st[4])
            elif st[0] == "delete":
                be.delete(st[1], st[2])
                rep.delete(st[1], st[2])
            elif st[0] == "lookup":
                continue
            elif st[0] == "drain":
                for m in harness.EVENT_MAPS:
                    be.drain(m)
                    rep.drain(m)
                continue
            else:
                if st[0] == "run_from":
                    d = st[2](want)
                    prog, arena, lens = st[1], d["arena"], d["lens"].astype(np.uint32)
                    off16, stride, now, prio, now_v = d.get("off16"), int(d.get("stride", 0)), int(d["now_ns"]), d.get("priority"), d.get("now_v")
                elif st[0] == "run":
                    _, prog, arena, lens, now, off16, stride, prio, now_v = st
                else:
                    raise AssertionError(st[0])
                outs = []
                for b in (be, rep):
                    a, l = arena.copy(), lens.copy()
                    p = None if prio is None else prio.copy()
                    v = b.run(prog, a, l, now, off16, stride, p, now_v) if now_v is not None else b.run(prog, a, l, now, off16, stride, p)
                    outs.append((np.asarray(v), a))
                assert np.array_equal(outs[0][0], want[tag + "_verdict"]), f"{script.name} {tag}: verdicts differ"
                assert np.array_equal(outs[0][1], want[tag + "_frames"]), f"{script.name} {tag}: frames differ"
            last = check_census(be.dp, _dumps(rep), f"{script.name} {tag}")
    finally:
        rep.close()
        be.close()
    return last


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("script", SCRIPTS)
def test_golden_scripts_census(script, pinned, ora_kind):
    last = run_census(scenarios.ALL_SCRIPTS[script], pinned, ora_kind)
    if script == "pipeline":
        # the reference allocator's collision hazard, pinned by real traffic (final tables of the pipeline golden)
        assert last[0]["sessions"] == 4802 and last[0]["unreachable"] == 279


@pytest.mark.parametrize("seed", [11, 13])
@pytest.mark.parametrize("prog", ["nat44_egress", "pipeline_up", "pipeline_tc"])
def test_fuzz_corpora_census(prog, seed, ora_kind):
    run_census(lambda: fuzz_script(prog, seed), False, ora_kind)


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("n", [255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049])
def test_batch_sizes_at_tile_and_chunk_edges(n, pinned, ora_kind, monkeypatch):
    monkeypatch.setenv("BNG_ZC_CHUNK_LOG2", "10")  # zero-copy chunks of 1024 frames (read at bng_open)
    run_census(_pipeline_batch(n), pinned, ora_kind)


# ---------------------------------------------------------------------------
# constructed tables
# ---------------------------------------------------------------------------
def _ip(a, b, c, d):
    return np.array([a, b, c, d], np.uint8)


def _addr(b):
    return int(np.asarray(b, np.uint8).view("<u4")[0])


def _sub_nat(dp, addr, pub, ps, pe, sub_id=1):
    v = np.zeros(1, L.subscriber_nat)
    v["block"]["public_ip"], v["block"]["port_start"], v["block"]["port_end"] = pub, ps, pe
    v["block"]["next_port"], v["block"]["subscriber_id"] = ps, sub_id
    assert dp.update("subscriber_nat", addr, v.view(np.uint8)) == 0


def _key(src, dst, sport, dport, proto):
    k = np.zeros(1, L.nat_key)
    k["src_ip"], k["dst_ip"], k["protocol"] = src, dst, proto
    k["src_port"] = np.array([sport >> 8, sport & 0xFF], np.uint8)
    k["dst_port"] = np.array([dport >> 8, dport & 0xFF], np.uint8)
    return k


def _session(dp, src, dst, sport, dport, proto, nat_ip, nat_port, reverse=True):
    k = _key(src, dst, sport, dport, proto)
    v = np.zeros(1, L.nat_session)
    v["nat_ip"], v["nat_port"] = nat_ip, np.array([nat_port >> 8, nat_port & 0xFF], np.uint8)
    v["orig_ip"], v["orig_port"], v["dest_ip"] = src, k["src_port"][0], dst
    v["dest_port"], v["protocol"], v["last_seen"], v["created"] = k["dst_port"][0], proto, 1, 1
    assert dp.update("nat_sessions", k.view(np.uint8), v.view(np.uint8)) == 0
    if reverse:
        rk = _key(dst, nat_ip, dport, nat_port, proto)
        assert dp.update("nat_reverse", rk.view(np.uint8), k.view(np.uint8)) == 0
    return k


def _eim(dp, internal, iport, proto, ext_ip, ext_port):
    k = np.zeros(1, L.eim_key)
    k["internal_ip"], k["internal_port"], k["protocol"] = internal, iport, proto
    v = np.zeros(1, L.eim_mapping)
    v["external_ip"], v["external_port"], v["ref_count"], v["last_used"] = ext_ip, ext_port, 1, 1
    assert dp.update("eim_table", k.view(np.uint8), v.view(np.uint8)) == 0


def _small():
    from bng_b200 import Dataplane
    return Dataplane(max_subscribers=1 << 10, max_nat_sessions=1 << 12, max_eim_mappings=1 << 12, max_batch=1 << 10)


def _by_addr(addrs, recs):
    return {int(a): r for a, r in zip(addrs, recs)}


def test_constructed_columns_eim_and_outside():
    A, B = _ip(10, 0, 0, 1), _ip(10, 0, 0, 2)
    P, Q = _ip(203, 0, 113, 1), _ip(203, 0, 113, 2)
    R = _ip(8, 8, 8, 8)
    with _small() as dp:
        _sub_nat(dp, A, P, 1000, 1009)  # 10 ports
        _sub_nat(dp, B, Q, 2000, 1999)  # port_end < port_start: no ports
        _session(dp, A, R, 5000, 80, 6, P, 1000)
        _session(dp, A, R, 5001, 80, 6, P, 1001)
        _session(dp, A, R, 5002, 53, 17, P, 1001)
        _session(dp, A, R, 5003, 0, 1, P, 1002)
        _session(dp, A, R, 5004, 9, 47, P, 1003)     # GRE: no column, counts in any
        _session(dp, A, R, 5005, 80, 6, P, 1010)     # outside: port past the block
        _session(dp, A, R, 5006, 80, 6, Q, 1000)     # outside: other public ip
        _eim(dp, A, 5007, 17, P, 1004)               # an EIM entry ...
        k = _session(dp, A, R, 5007, 443, 17, P, 1004)  # ... and its session hold one triple
        _session(dp, A, _ip(9, 9, 9, 9), 5007, 443, 17, P, 1004)
        got = check_census(dp, _dumps(dp), "constructed")
        s, sa, sr, pa, pr = got
        sub = _by_addr(sa, sr)[_addr(A)]
        assert sub["in_use"].tolist() == [2, 2, 1] and sub["in_use_any"] == 5 and sub["outside"] == 2
        assert sub["sessions"] == 9 and sub["eim"] == 1 and sub["block_ports"] == 10 and sub["permille"] == 200
        assert _by_addr(sa, sr)[_addr(B)]["block_ports"] == 0 and _by_addr(sa, sr)[_addr(B)]["permille"] == 0
        pub = _by_addr(pa, pr)
        assert pub[_addr(P)]["in_use"].tolist() == [3, 2, 1] and pub[_addr(P)]["in_use_any"] == 6
        assert pub[_addr(P)]["blocks"] == 1 and pub[_addr(Q)]["blocks"] == 1 and pub[_addr(Q)]["sessions"] == 1
        assert s["triples"] == 8 and s["unreachable"] == 0 and s["stale_reverse"] == 0
        assert k["protocol"][0] == 17


def test_constructed_unreachable_stale_orphans_and_moves():
    A, B = _ip(10, 0, 0, 1), _ip(10, 0, 0, 2)
    P = _ip(203, 0, 113, 1)
    R = _ip(8, 8, 8, 8)
    with _small() as dp:
        _sub_nat(dp, A, P, 1000, 1999)
        _sub_nat(dp, B, P, 1000, 1999)  # overlapping blocks: both hand out the same ports
        _session(dp, A, R, 4000, 80, 6, P, 1500)
        _session(dp, B, R, 4001, 80, 6, P, 1500)  # the same port and remote: its reverse entry replaces A's
        _session(dp, A, R, 4002, 80, 6, P, 1501, reverse=False)  # no reverse entry at all
        stale = _key(R, P, 80, 1999, 6)
        assert dp.update("nat_reverse", stale.view(np.uint8), _key(A, R, 4999, 80, 6).view(np.uint8)) == 0
        s = check_census(dp, _dumps(dp), "hazard")[0]
        assert s["unreachable"] == 2 and s["stale_reverse"] == 1 and s["triples"] == 2
        # the block moves: the sessions stay and are now outside it
        _sub_nat(dp, A, _ip(203, 0, 113, 9), 1000, 1999)
        s, sa, sr, _, _ = check_census(dp, _dumps(dp), "moved")
        assert _by_addr(sa, sr)[_addr(A)]["outside"] == 2 and _by_addr(sa, sr)[_addr(A)]["in_use"][0] == 0
        # released without a flush: orphans
        assert dp.delete("subscriber_nat", A) == 0
        _eim(dp, A, 4000, 6, P, 1500)
        s = check_census(dp, _dumps(dp), "orphans")[0]
        assert s["orphan_sessions"] == 2 and s["orphan_eim"] == 1 and s["subscribers"] == 1


def test_constructed_block_extremes_addresses_and_caps():
    A, B, C = _ip(10, 0, 0, 1), _ip(10, 0, 0, 2), _ip(10, 0, 0, 3)
    Z, F = _ip(0, 0, 0, 0), _ip(255, 255, 255, 255)
    R = _ip(8, 8, 8, 8)
    with _small() as dp:
        _sub_nat(dp, A, Z, 7, 7)          # one port, on public address 0
        _sub_nat(dp, B, F, 0, 65535)      # every port, on 255.255.255.255
        _sub_nat(dp, C, F, 100, 103)
        _session(dp, A, R, 1, 80, 6, Z, 7)
        for p in range(3):
            _session(dp, B, R, 100 + p, 80, 17, F, 60000 + p)
        _session(dp, C, R, 1, 80, 6, F, 100)
        _session(dp, C, R, 2, 80, 6, F, 101)
        want = check_census(dp, _dumps(dp), "extremes")
        pm = {int(a): int(r["permille"]) for a, r in zip(want[1], want[2])}
        assert pm == {_addr(A): 1000, _addr(B): 0, _addr(C): 500}
        assert set(want[3].tolist()) == {_addr(Z), _addr(F)}
        assert _by_addr(want[3], want[4])[_addr(F)]["block_ports"] == 65536 + 4
        # min_permille exactly at a record's permille qualifies it
        for mp, names in ((500, {_addr(A), _addr(C)}), (501, {_addr(A)}), (1000, {_addr(A)})):
            check_census(dp, _dumps(dp), f"min {mp}", mp)
            assert set(dp.nat_usage(mp)[1].tolist()) == names
        # caps below found: min(found, cap) records, found reported in full
        s, sa, sr, pa, pr = dp.nat_usage(0, cap=1)
        assert s["subs_found"] == 3 and s["pubs_found"] == 2 and len(sa) == 1 and len(pa) == 1
        full = _by_addr(want[1], want[2])
        assert sr[0].tobytes() == full[int(sa[0])].tobytes()
        s0 = dp.nat_usage(0, cap=0)
        assert s0[0] == s and len(s0[1]) == 0 and len(s0[3]) == 0


def test_many_public_addresses_grow_the_table():
    """More public addresses than the first public-address table holds: the census grows it and stays exact."""
    from bng_b200 import Dataplane
    n = 40_000
    with Dataplane(max_subscribers=1 << 10, max_nat_sessions=1 << 16, max_eim_mappings=1 << 10, max_batch=1 << 10) as dp:
        _sub_nat(dp, _ip(10, 0, 0, 1), _ip(203, 0, 113, 1), 1000, 1999)
        i = np.arange(n, dtype=np.uint32)
        k = np.zeros(n, L.nat_key)
        k["src_ip"] = _ip(10, 0, 0, 1)
        k["dst_ip"] = _ip(8, 8, 8, 8)
        k["src_port"][:, 0], k["src_port"][:, 1] = i >> 8, i & 0xFF
        k["protocol"] = 17
        v = np.zeros(n, L.nat_session)
        v["nat_ip"] = np.ascontiguousarray((0x0A000000 + i).astype(">u4")).view(np.uint8).reshape(-1, 4)
        v["nat_port"] = np.array([4, 0], np.uint8)
        v["protocol"] = 17
        assert dp.update_batch("nat_sessions", k.view(np.uint8).reshape(n, -1), v.view(np.uint8).reshape(n, -1)) == 0
        s = check_census(dp, _dumps(dp), "40k public addresses")[0]
        assert s["pubs_found"] == n + 1 and s["unreachable"] == n
        assert check_census(dp, _dumps(dp), "again")[0] == s


# ---------------------------------------------------------------------------
# churn
# ---------------------------------------------------------------------------
def test_churn_sweep_flush_eviction_rebuild_staged_clear():
    from bng_b200 import Dataplane
    n_subs = 6
    with Dataplane(max_subscribers=64, max_nat_sessions=256, max_eim_mappings=256, max_batch=1 << 12) as dp:
        sc = harness.Script("setup")
        scenarios.nat_maps(sc, n_subs, 64, 0x0F)
        for st in sc.steps:
            assert dp.update_batch(st[1], st[2], st[3]) == 0
        keys = S.ip_bytes(S.sub_ip(np.arange(n_subs)))
        r = np.random.Generator(np.random.PCG64(7))
        for step in range(14):
            n = 700
            sub = r.integers(0, n_subs, n)
            sport = (10000 + step * 1000 + r.integers(0, 900, n)).astype(np.uint32)
            lens = np.full(n, 64, np.uint32)
            proto = np.where(r.integers(0, 2, n) == 0, 6, 17).astype(np.uint32)
            hdr = S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), np.full(n, 0x08080808, np.uint32),
                                 proto, sport, np.full(n, 53, np.uint32), lens)
            dp.run("nat44_egress", hdr.reshape(-1).copy(), lens, (step + 1) * 10**9, stride=64)
            if step == 4:
                dp.sweep(10**13)
            if step == 7:
                dp.nat_flush(keys[:2], 8 * 10**9)
            if step == 10:  # staged upserts pending at the call: the census applies them first
                v = np.zeros(1, L.subscriber_nat)
                v["block"]["public_ip"], v["block"]["port_start"], v["block"]["port_end"] = _ip(198, 51, 100, 7), 100, 163
                assert dp.update_staged("subscriber_nat", _ip(10, 9, 9, 9), v.view(np.uint8)) == 0
            check_census(dp, _dumps(dp), f"step {step}")
        assert dp.lru_evictions > 0 and dp.table_rebuilds > 0
        for m in ("nat_sessions", "eim_table", "nat_reverse"):
            dp.clear(m)
        s = check_census(dp, _dumps(dp), "cleared")[0]
        assert s["sessions"] == s["eim"] == s["triples"] == 0 and s["subscribers"] == n_subs + 1


# ---------------------------------------------------------------------------
# read-only
# ---------------------------------------------------------------------------
def _pipeline_run(census):
    """The pipeline golden script on one context with accounting, idle stamps and delta tracking on; census=True adds
    a census after every step.  Returns what the script leaves behind and the program runs' launch counts."""
    from bng_b200 import Dataplane
    script = scenarios.ALL_SCRIPTS["pipeline"]()
    out = {"launches": [], "verdicts": [], "events": []}
    with Dataplane(max_subscribers=1 << 14, max_nat_sessions=1 << 16, max_eim_mappings=1 << 16, max_batch=1 << 16,
                   event_capacity=1 << 16) as dp:
        for p in ("pipeline_up", "nat44_ingress"):
            dp.acct_enable(p)
            dp.idle_enable(p)
        dp.delta_enable()
        dp.delta_export()
        for st in script.steps:
            if st[0] == "update":
                dp.update_batch(st[1], st[2], st[3], st[4])
            elif st[0] == "delete":
                dp.delete(st[1], st[2])
            elif st[0] == "drain":
                out["events"].append([dp.drain(m) for m in harness.EVENT_MAPS])
            elif st[0] == "run":
                _, prog, arena, lens, now, off16, stride, prio, now_v = st
                c0 = dp.launch_count
                v = dp.run(prog, arena.copy(), lens.copy(), now, off16=off16, stride=stride, priority=None if prio is None else prio.copy(),
                           now_v=now_v)
                out["launches"].append(dp.launch_count - c0)
                out["verdicts"].append(np.asarray(v).copy())
                dp.delta_export()  # the run's changes
                if census:
                    c1 = dp.launch_count
                    dp.nat_usage()
                    dp.nat_usage(300)
                    assert dp.launch_count > c1
                    assert _delta_changes(dp.delta_export()) == 0, "a census left changes for the standby"
        out["events"].append([dp.drain(m) for m in harness.EVENT_MAPS])
        out["tables"] = {m: dp.dump(m) for m in harness.TABLES}
        out["stats"] = {m: dp.stats(m) for m in harness.STATS_MAPS}
        out["acct"] = dp.acct_dump()
        addrs = out["acct"][0]
        out["idle"] = dp.idle_read(addrs)
        out["idle_scan"] = dp.idle_scan(10**12)
    return out


def _delta_changes(blob):
    """Deleted and upserted entries of the sections that carry changes only (hash maps, accounting, interception
    targets, idle timeouts); array, LPM and statistics maps are sent whole every time."""
    _, sections = L.parse_delta(blob)
    return sum(len(dk) + len(uk) for kind, dk, uk, _ in sections.values() if kind in (0, 5, 6, 7))


def _same(a, b, what):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _same(a[k], b[k], f"{what}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{what}[{i}]")
    elif isinstance(a, np.ndarray):
        assert np.array_equal(a, b), what
    else:
        assert a == b, what


def test_census_is_read_only():
    plain, with_census = _pipeline_run(False), _pipeline_run(True)
    _same(plain, with_census, "pipeline with and without censuses")


# ---------------------------------------------------------------------------
# scale, sharding, errors
# ---------------------------------------------------------------------------
def test_cold_nat_at_reference_capacities():
    from bng_b200 import Dataplane
    n = 1 << 22
    wl = W.build("nat_cold_64", n, subs_scale=4)  # 65 536 subscribers x 64 flows: 2^22 new flows
    assert wl.n == n
    with Dataplane(max_batch=n) as dp:
        for m, k, v in wl.maps:
            assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
        for prog, h, l in wl.prewarm:
            dp.run(prog, h.reshape(-1).copy(), l.copy(), wl.now0 - 1, stride=64)
        dp.run(wl.prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0, stride=64)
        s = check_census(dp, _dumps(dp), "nat_cold_64 2^22")[0]
        assert s["sessions"] > 3_000_000 and s["subscribers"] == 65536


def merge_censuses(parts):
    """Router::NatUsage's merge: summaries summed, subscriber records from their owner shards, public-address records
    summed by address (a triple held on two shards counts once per shard)."""
    summary = {k: sum(p[0][k] for p in parts) for k in parts[0][0]}
    sa = np.concatenate([p[1] for p in parts])
    sr = np.concatenate([p[2] for p in parts])
    pubs = {}
    for p in parts:
        for a, r in zip(p[3].tolist(), p[4]):
            if a in pubs:
                acc = pubs[a]
                for f in L.bng_nat_pub_use.names:
                    acc[f] = acc[f] + r[f]
            else:
                pubs[a] = r.copy()
    pa = np.array(sorted(pubs, key=lambda a: np.array([a], "<u4").byteswap()[0]), "<u4")
    pr = np.array([pubs[int(a)] for a in pa], L.bng_nat_pub_use) if len(pa) else np.zeros(0, L.bng_nat_pub_use)
    summary["pubs_found"] = len(pa)
    o = np.argsort(sa.byteswap(), kind="stable")
    return summary, sa[o], sr[o], pa, pr


@pytest.mark.parametrize("world", [2, 8])
def test_sharded_census_merges_to_the_unsharded_one(world):
    from bng_b200 import Dataplane
    n, n_subs = 1 << 16, 1_000
    wl = W.pipeline(n, 0, 1, n_subs=n_subs, flows_per_sub=16, imix=True)
    sub = np.arange(n_subs, dtype=np.uint32)
    ip_shard = {bytes(k): int(s) for k, s in zip(S.ip_bytes(S.sub_ip(sub)), S.shard_of_mac(S.sub_mac_key(sub), world))}

    def macs(h):
        mac = np.zeros(len(h), np.uint64)
        for i in range(6):
            mac = (mac << np.uint64(8)) | h[:, 6 + i].astype(np.uint64)
        return mac

    frame_shard = S.shard_of_mac(macs(wl.headers), world)
    warm_h, warm_l = wl.prewarm[0][1], wl.prewarm[0][2]
    warm_shard = S.shard_of_mac(macs(warm_h), world)

    def run(rank, world_):
        dp = Dataplane(max_batch=n, max_subscribers=4 * n_subs + 1024, max_nat_sessions=1 << 18, max_eim_mappings=1 << 18)
        try:
            for m, k, v in wl.maps:
                kb, vb = as_bytes(k), as_bytes(v)
                if world_ > 1 and m in ("subscriber_nat", "qos_ingress"):
                    keep = np.array([ip_shard[bytes(x)] == rank for x in kb])
                    kb, vb = kb[keep], vb[keep]
                elif world_ > 1 and m == "subscriber_bindings":
                    keep = S.shard_of_mac(k.astype(np.uint64), world_) == rank
                    kb, vb = kb[keep], vb[keep]
                assert dp.update_batch(m, kb, vb) == 0, m
            mw = (warm_shard == rank) if world_ > 1 else np.ones(len(warm_h), bool)
            dp.run("nat44_egress", warm_h[mw].reshape(-1).copy(), warm_l[mw].copy(), wl.now0 - 1, stride=64)
            mine = np.nonzero(frame_shard == rank)[0] if world_ > 1 else np.arange(n)
            for s in range(2):
                dp.run(wl.prog, wl.headers[mine].reshape(-1).copy(), wl.lens[mine].copy(), wl.now0 + s * wl.now_step, stride=64)
            check_census(dp, _dumps(dp), f"shard {rank}/{world_}")
            return dp.nat_usage()
        finally:
            dp.close()

    whole = run(0, 1)
    merged = merge_censuses([run(r, world) for r in range(world)])
    assert whole[0]["sessions"] > 0
    _same(merged[0], whole[0], "summary")
    for i in (1, 2, 3, 4):
        assert merged[i].tobytes() == whole[i].tobytes(), f"merged census part {i} differs"


def test_error_codes():
    from bng_b200 import BngError
    with _small() as dp:
        lib, h = dp.lib, dp.h
        s = np.zeros(1, L.bng_nat_usage_sum)
        a = np.zeros(4, "<u4")
        r = np.zeros(4, L.bng_nat_sub_use)
        p = np.zeros(4, L.bng_nat_pub_use)
        ok = (s.ctypes.data, a.ctypes.data, r.ctypes.data, 4, a.ctypes.data, p.ctypes.data, 4)
        assert lib.bng_nat_usage(h, 0, *ok) == 0
        assert lib.bng_nat_usage(None, 0, *ok) == -errno.EINVAL
        assert lib.bng_nat_usage(h, 0, None, *ok[1:]) == -errno.EINVAL
        assert lib.bng_nat_usage(h, 1001, *ok) == -errno.EINVAL
        assert lib.bng_nat_usage(h, 1000, *ok) == 0
        assert lib.bng_nat_usage(h, 0, s.ctypes.data, None, r.ctypes.data, 1, a.ctypes.data, p.ctypes.data, 4) == -errno.EINVAL
        assert lib.bng_nat_usage(h, 0, s.ctypes.data, a.ctypes.data, None, 1, a.ctypes.data, p.ctypes.data, 4) == -errno.EINVAL
        assert lib.bng_nat_usage(h, 0, s.ctypes.data, a.ctypes.data, r.ctypes.data, 4, None, p.ctypes.data, 1) == -errno.EINVAL
        assert lib.bng_nat_usage(h, 0, s.ctypes.data, a.ctypes.data, r.ctypes.data, 4, a.ctypes.data, None, 1) == -errno.EINVAL
        assert lib.bng_nat_usage(h, 0, s.ctypes.data, None, None, 0, None, None, 0) == 0
        with pytest.raises(BngError) as e:
            dp.nat_usage(1001)
        assert e.value.errno == errno.EINVAL
