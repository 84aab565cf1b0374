"""Subscriber hand-over between contexts (bng_sub_export / bng_sub_import) on the GPU.

The mid-stream move runs two shards as test_gpu_sharded does, moves a third of shard 0's subscribers to shard 1
between batches, steers the later frames by the new owners, and holds the union of the shards against one reference
run over the same frames and, for the GPU-only state (accounting, idle records, interception), against one context
that never moved anything.  The other tests pin down the export's selection, the round trip, the error paths and the
interplay with delta replication."""
import numpy as np
import pytest

import harness
from bng_b200 import layouts as L
from bng_b200 import synth as S
from bng_b200 import workloads as W
from bng_b200.layouts import as_bytes

pytestmark = pytest.mark.gpu

NS = 10**9
STATS = ("antispoof_stats", "qos_stats_map", "nat_stats_map")
FLOW = ("nat_sessions", "nat_reverse", "eim_table")
TABLES = FLOW + ("subscriber_nat", "qos_ingress", "qos_egress", "subscriber_bindings", "subscriber_pools")
KEYED_BY_SUBSCRIBER = {"subscriber_bindings": "mac", "subscriber_pools": "mac", "qos_ingress": "ip", "qos_egress": "ip",
                       "subscriber_nat": "ip"}
EINVAL, ENOSPC, E2BIG = 22, 28, 7


def _words(b):
    return np.ascontiguousarray(b).view("<u4").reshape(-1)


def _mac_keys(h):
    k = np.zeros(len(h), np.uint64)
    for i in range(6):
        k = (k << np.uint64(8)) | h[:, 6 + i].astype(np.uint64)
    return k


def _rows(name, k, v):
    if len(k) == 0:
        return []
    return sorted(bytes(r) for r in np.concatenate([k, harness.mask_padding(name, v)], axis=1))


def parse_blob(blob):
    """{section name: (keys u8[n, ks], values u8[n, vs])} and the offsets where sections start."""
    assert blob[:8] == b"BNGMOVE1"
    secs = harness.blob_sections(blob)
    return {s.name: (s.keys, s.vals) for s in secs}, [s.start for s in secs]


def _state(dp):
    """Every map a subscriber owns, the accounting and idle records and the interception targets (as a read-only
    export of every address sees them), each as a sorted row list."""
    st = {m: _rows(m, *dp.dump(m)) for m in TABLES}
    a, rec = dp.acct_dump()
    st["acct"] = sorted(zip(a.tolist(), [bytes(r) for r in rec.view(np.uint8).reshape(len(a), 64)]))
    if len(a):
        ir, found = dp.idle_read(a)
        st["idle"] = sorted(zip(a[found].tolist(), [bytes(r) for r in ir[found].view(np.uint8).reshape(-1, 32)]))
    li = parse_blob(dp.sub_export(_words(dp.dump("subscriber_nat")[0])))[0].get("li_targets")
    st["li"] = _rows("li", *li) if li is not None else []
    return st


def _load(dp, wl, keep_ip=None, keep_mac=None):
    for m, k, v in wl.maps:
        kb, vb = as_bytes(k), as_bytes(v)
        how = KEYED_BY_SUBSCRIBER.get(m)
        if how == "mac" and keep_mac is not None:
            sel = keep_mac(k.astype(np.uint64))
            kb, vb = kb[sel], vb[sel]
        elif how == "ip" and keep_ip is not None:
            sel = keep_ip(_words(kb))
            kb, vb = kb[sel], vb[sel]
        assert dp.update_batch(m, kb, vb) == 0, m


# ---------------------------------------------------------------------------
# 1 + 2: a mid-stream move equals the unsharded reference and a context that never moved
# ---------------------------------------------------------------------------
N, N_SUBS, STEPS = 1 << 17, 2_000, 2


def _replies(sessions, n_max=4096):
    """nat44_ingress frames answering UDP sessions of a nat_sessions dump: remote -> (nat_ip, nat_port)."""
    k, v = sessions
    vv = v.copy().view(L.nat_session).reshape(-1)
    pick = np.nonzero(vv["protocol"] == 17)[0][:n_max]
    h = S.ipv4_headers(np.uint64(0x02FFFFFFFFFE), np.uint64(0x020000000001), 0, 0, 17, 0, 0, 64)
    h = np.repeat(h, len(pick), axis=0)
    h[:, 26:30] = k[pick, 4:8]      # the session key's dst_ip / dst_port, network order
    h[:, 34:36] = k[pick, 10:12]
    h[:, 30:34] = v[pick, 0:4]      # nat_ip, nat_port (network order)
    h[:, 36:38] = v[pick, 4:6]
    return h, np.full(len(pick), 64, np.uint32)


def _block_owner(subnat, replies):
    """The subscriber address (u32 key word) holding the port block each reply is addressed to."""
    k, v = subnat
    b = v.copy().view(L.subscriber_nat).reshape(-1)["block"]
    pub = _words(b["public_ip"].copy())
    port = (replies[:, 36].astype(np.uint32) << 8) | replies[:, 37]
    dst = _words(replies[:, 30:34].copy())
    out = np.zeros(len(replies), "<u4")
    ipw = _words(k)
    for i in range(len(replies)):
        hit = np.nonzero((pub == dst[i]) & (b["port_start"] <= port[i]) & (b["port_end"] >= port[i]))[0]
        assert len(hit) == 1
        out[i] = ipw[hit[0]]
    return out


def _li_rows(hdr, caps, frame_of):
    """Per target: (run, global frame, the record without batch / frame, captured bytes), in frame order."""
    per = {}
    for h, c in zip(hdr, caps):
        run, g = frame_of(int(h["batch"]), int(h["frame"]))
        r = h.copy()
        r["batch"], r["frame"] = 0, 0
        per.setdefault(int(h["target_id"]), []).append((run, g, r.tobytes(), bytes(c)))
    return {t: sorted(v) for t, v in per.items()}


@pytest.mark.parametrize("prog", ["pipeline_up", "pipeline_tc"])
def test_mid_stream_move_equals_the_unsharded_reference(prog):
    from bng_b200 import Dataplane
    from oracle.pyoracle import Oracle, available
    wl = W.pipeline(N, 0, 1, n_subs=N_SUBS, flows_per_sub=16, imix=True)
    world = 2
    sub = np.arange(N_SUBS)
    sub_ipw = _words(S.ip_bytes(S.sub_ip(sub)))
    sub_mac = S.sub_mac_key(sub)
    home = S.shard_of_mac(sub_mac, world).astype(np.int64)
    frame_sub = (_mac_keys(wl.headers) & np.uint64(0xFFFFFFFF)).astype(np.int64)
    warm_h, warm_l = wl.prewarm[0][1], wl.prewarm[0][2]
    warm_sub = (_mac_keys(warm_h) & np.uint64(0xFFFFFFFF)).astype(np.int64)
    # a third of shard 0's subscribers, the ten with the most frames among them
    on0 = np.nonzero(home == 0)[0]
    fat = on0[np.argsort(-np.bincount(frame_sub, minlength=N_SUBS)[on0], kind="stable")]
    moved = np.unique(np.concatenate([fat[:10], fat[10::3]]))
    owner = home.copy()
    owner[moved] = 1
    li_addrs = np.concatenate([sub_ipw[moved[:3]], sub_ipw[on0[~np.isin(on0, moved)][:2]], sub_ipw[home == 1][:2]])
    timeouts = (sub % 7 * 60 + 30).astype("<u4")

    # the reference: one run over every frame
    o = Oracle("reference" if available("reference") else "port")
    for m, k, v in wl.maps:
        assert o.update_batch(m, as_bytes(k), as_bytes(v)) == 0
    pa = o.arena(warm_h.shape[0] * 64 + 64)
    pa[: warm_h.shape[0] * 64] = warm_h.reshape(-1)
    o.run("nat44_egress", pa, warm_l.copy(), wl.now0 - 1, stride=64)
    for m in ("spoof_events", "nat_log_rb"):
        o.drain(m)
    ref = []
    for s in range(2 * STEPS):
        oa = o.arena(wl.n * 64 + 64)
        oa[: wl.n * 64] = wl.headers.reshape(-1)
        v = o.run(prog, oa, wl.lens.copy(), wl.now0 + s * wl.now_step, stride=64)
        ref.append((np.asarray(v).copy(), np.array(oa[: wl.n * 64]).reshape(-1, 64)))
        o.free_arenas()
    rep_h, rep_l = _replies(o.dump("nat_sessions"))
    rep_owner_ip = _block_owner(o.dump("subscriber_nat"), rep_h)
    t_rep = wl.now0 + 2 * STEPS * wl.now_step
    oa = o.arena(len(rep_h) * 64 + 64)
    oa[: len(rep_h) * 64] = rep_h.reshape(-1)
    v = o.run("nat44_ingress", oa, rep_l.copy(), t_rep, stride=64)
    ref.append((np.asarray(v).copy(), np.array(oa[: len(rep_h) * 64]).reshape(-1, 64)))
    o.free_arenas()
    ref_stats = {m: o.lookup(m, np.zeros(4, np.uint8)).view("<u8").copy() for m in STATS}
    ref_events = {m: o.drain(m) for m in ("spoof_events", "nat_log_rb")}
    ref_tables = {m: _rows(m, *o.dump(m)) for m in TABLES}
    ip_home = dict(zip(sub_ipw.tolist(), home.tolist()))
    ip_owner = dict(zip(sub_ipw.tolist(), owner.tolist()))
    assert any(ip_owner[a] == 1 and a in set(sub_ipw[moved].tolist()) for a in rep_owner_ip.tolist())
    assert any(ip_owner[a] == 0 for a in rep_owner_ip.tolist())

    def features(dp, addrs):
        for p in (prog, "nat44_ingress"):
            dp.acct_enable(p)
            dp.idle_enable(p)
        mine = np.isin(sub_ipw, addrs)
        assert dp.idle_timeout_set(sub_ipw[mine], timeouts[mine]).all()
        for i, a in enumerate(li_addrs.tolist()):
            if a in set(addrs.tolist()):
                dp.li_target_set(a, 100 + i)

    opts = dict(max_batch=N, max_subscribers=4 * N_SUBS, max_nat_sessions=1 << 18, max_eim_mappings=1 << 18)
    # the context that never moved anything: every frame, every subscriber
    one = Dataplane(**opts)
    try:
        _load(one, wl)
        features(one, sub_ipw)
        one.run("nat44_egress", warm_h.reshape(-1).copy(), warm_l.copy(), wl.now0 - 1, stride=64)
        for s in range(2 * STEPS):
            one.run(prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0 + s * wl.now_step, stride=64)
        one.run("nat44_ingress", rep_h.reshape(-1).copy(), rep_l.copy(), t_rep, stride=64)
        one_acct = one.acct_dump()
        one_idle = one.idle_read(one_acct[0])
        one_li = one.li_drain()
    finally:
        one.close()

    # two shards; the move happens after STEPS batches
    dps = [Dataplane(rank=r, world=world, **opts) for r in range(world)]
    got = [(np.full(N, 255, np.uint8), np.zeros((N, 64), np.uint8)) for _ in range(2 * STEPS)]
    got.append((np.full(len(rep_h), 255, np.uint8), np.zeros((len(rep_h), 64), np.uint8)))
    index = [[None] * (2 * STEPS + 2) for _ in range(world)]  # per shard and run: global frame of each shard frame
    events = {m: [] for m in ref_events}
    try:
        for r, dp in enumerate(dps):
            _load(dp, wl, keep_ip=lambda w, r=r: np.array([ip_home.get(int(x)) == r for x in w], bool),
                  keep_mac=lambda k, r=r: S.shard_of_mac(k, world) == r)
            features(dp, sub_ipw[home == r])
            mine = np.nonzero(home[warm_sub] == r)[0]
            index[r][0] = mine
            dp.run("nat44_egress", warm_h[mine].reshape(-1).copy(), warm_l[mine].copy(), wl.now0 - 1, stride=64)
            for m in ("spoof_events", "nat_log_rb"):
                dp.drain(m)
        for s in range(2 * STEPS):
            if s == STEPS:  # the hand-over, between two batches
                for dp in dps:
                    events["nat_log_rb"].append(dp.drain("nat_log_rb"))
                blob = dps[0].sub_export(sub_ipw[moved], sub_mac[moved], detach=True)
                assert dps[1].sub_import(blob) == 0
                assert all(len(dp.drain("nat_log_rb")) == 0 for dp in dps), "the move logged something"
            own = home if s < STEPS else owner
            for r, dp in enumerate(dps):
                mine = np.nonzero(own[frame_sub] == r)[0]
                index[r][1 + s] = mine
                a = wl.headers[mine].reshape(-1).copy()
                got[s][0][mine] = dp.run(prog, a, wl.lens[mine].copy(), wl.now0 + s * wl.now_step, stride=64)
                got[s][1][mine] = a.reshape(-1, 64)
        rep_shard = np.array([ip_owner[int(a)] for a in rep_owner_ip])
        for r, dp in enumerate(dps):
            mine = np.nonzero(rep_shard == r)[0]
            index[r][-1] = mine
            a = rep_h[mine].reshape(-1).copy()
            got[-1][0][mine] = dp.run("nat44_ingress", a, rep_l[mine].copy(), t_rep, stride=64)
            got[-1][1][mine] = a.reshape(-1, 64)
        stats = {m: sum(dp.stats(m).astype(np.uint64) for dp in dps) for m in STATS}
        for m in events:
            events[m].extend(dp.drain(m) for dp in dps)
        tables = {m: sorted(sum((_rows(m, *dp.dump(m)) for dp in dps), [])) for m in TABLES}
        acct = [dp.acct_dump() for dp in dps]
        idle = [dp.idle_read(a[0]) for dp, a in zip(dps, acct)]
        lis = [dp.li_drain() for dp in dps]
        assert all(dp.lru_overflow == 0 and dp.events_lost == 0 for dp in dps)
    finally:
        for dp in dps:
            dp.close()

    for s, (v, f) in enumerate(ref):
        assert np.array_equal(got[s][0], v), f"run {s}: verdicts differ"
        assert np.array_equal(got[s][1], f), f"run {s}: frame bytes differ"
    for m in STATS:
        assert np.array_equal(stats[m], ref_stats[m]), f"{m}: {stats[m]} vs {ref_stats[m]}"
    for m, parts in events.items():
        g = np.concatenate([p for p in parts if len(p)], axis=0) if any(len(p) for p in parts) else np.zeros((0, 1), np.uint8)
        want = ref_events[m]
        w = (g.shape[1] if len(g) else want.shape[1]) - (4 if m == "nat_log_rb" else 0)
        assert sorted(bytes(r) for r in g[:, :w]) == sorted(bytes(r) for r in want[:, :w]), f"{m}: event multisets differ"
    for m in TABLES:
        assert tables[m] == ref_tables[m], f"{m}: union of the shards differs from the reference"
    # GPU-only state: the union of the shards is the unmoved context's
    ua = np.concatenate([a[0] for a in acct])
    ur = np.concatenate([a[1] for a in acct])
    ui = np.concatenate([i[0] for i in idle])
    assert all(i[1].all() for i in idle)
    o_ = np.argsort(ua, kind="stable")
    oa_ = np.argsort(one_acct[0], kind="stable")
    assert np.array_equal(ua[o_], one_acct[0][oa_]) and np.array_equal(ur[o_], one_acct[1][oa_]), "accounting records differ"
    assert np.array_equal(ui[o_], one_idle[0][oa_]), "idle records differ"
    assert (ui["flags"] & L.IDLE_UP).any() and (ui["flags"] & L.IDLE_DOWN).any()

    def shard_frame(r):
        return lambda batch, frame: (batch - 1, int(index[r][batch - 1][frame]))
    got_li = {}
    for r, (h, c) in enumerate(lis):
        for t, rows in _li_rows(h, c, shard_frame(r)).items():
            got_li.setdefault(t, []).extend(rows)
    want_li = _li_rows(one_li[0], one_li[1], lambda batch, frame: (batch - 1, frame))
    assert {t: sorted(v) for t, v in got_li.items()} == want_li, "interception records differ"
    assert len(want_li) == len(li_addrs) and all(len(v) for v in want_li.values())


# ---------------------------------------------------------------------------
# 3 - 10 on smaller contexts
# ---------------------------------------------------------------------------
SMALL = dict(max_batch=1 << 14, max_subscribers=1 << 11, max_nat_sessions=1 << 14, max_eim_mappings=1 << 14)


def _small(opts=SMALL, n_subs=400):
    """A context with pipeline_up state for n_subs subscribers, accounting, idle records and two LI targets."""
    from bng_b200 import Dataplane
    wl = W.pipeline(1 << 13, 0, 1, n_subs=n_subs, flows_per_sub=8, imix=True)
    dp = Dataplane(**opts)
    _load(dp, wl)
    dp.acct_enable("pipeline_up")
    dp.idle_enable("pipeline_up")
    ips = _words(S.ip_bytes(S.sub_ip(np.arange(n_subs))))
    dp.idle_timeout_set(ips, 300)
    dp.li_target_set(int(ips[1]), 7)
    dp.li_target_set(int(ips[5]), 8)
    for p, h, l in wl.prewarm:
        dp.run(p, h.reshape(-1).copy(), l.copy(), wl.now0 - 1, stride=64)
    dp.run("pipeline_up", wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0, stride=64)
    dp.drain("nat_log_rb")
    dp.drain("spoof_events")
    return dp, wl, ips


def _sections_equal(a, b):
    pa, pb = parse_blob(a)[0], parse_blob(b)[0]
    assert pa.keys() == pb.keys()
    for m in pa:
        assert _rows(m, *pa[m]) == _rows(m, *pb[m]), m


def test_round_trip_and_read_only_export():
    dp, wl, ips = _small()
    twin = _small()[0]
    try:
        addrs = ips[1::4]  # both interception targets among them
        macs = S.sub_mac_key(np.arange(len(ips))[1::4])
        before = _state(dp)
        ro = dp.sub_export(addrs, macs)
        assert _state(dp) == before, "a read-only export changed the context"
        blob = dp.sub_export(addrs, macs, detach=True)
        _sections_equal(ro, blob)
        sec = parse_blob(blob)[0]
        assert all(len(sec[m][0]) for m in FLOW + ("subscriber_nat", "subscriber_bindings", "subscriber_acct",
                                                    "subscriber_idle_rec", "li_targets"))
        assert _state(dp) != before
        assert dp.sub_import(blob) == 0
        assert _state(dp) == before, "the round trip did not restore the context"
        # the next batch: the same outputs as a context that never moved anything
        outs = []
        for c in (dp, twin):
            a = wl.headers.reshape(-1).copy()
            v = c.run("pipeline_up", a, wl.lens.copy(), wl.now0 + wl.now_step, stride=64)
            outs.append((v.copy(), a.copy(), _state(c), c.drain("nat_log_rb")))
        assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
        assert outs[0][2] == outs[1][2]
        assert sorted(bytes(r) for r in outs[0][3]) == sorted(bytes(r) for r in outs[1][3])
    finally:
        dp.close()
        twin.close()


def test_exact_selection():
    dp, wl, ips = _small()
    try:
        members = ips[::5]
        nobody = np.array([0x0A0B0C0D], "<u4")  # an address without state
        # a member's stale reverse entry, and a non-member's session towards a member's address
        k, v = dp.dump("nat_reverse")
        stale_k = k[0].copy()
        stale_k[8:10] = [0xEE, 0xEE]
        stale_v = np.zeros(16, np.uint8)
        stale_v[0:4] = members[0:1].view(np.uint8)
        assert dp.update("nat_reverse", stale_k, stale_v) == 0
        sk, sv = dp.dump("nat_sessions")
        src = _words(sk[:, 0:4].copy())
        i = int(np.nonzero(~np.isin(src, members))[0][0])
        odd_k = sk[i].copy()
        odd_k[4:8] = members[1:2].view(np.uint8)
        assert dp.update("nat_sessions", odd_k, sv[i]) == 0
        macs = S.sub_mac_key(np.arange(len(ips))[::5])
        before = {m: dp.dump(m) for m in TABLES}
        addrs = np.concatenate([members, nobody, members[:3]])  # repeats are harmless
        blob = dp.sub_export(addrs, np.concatenate([macs, macs[:2]]), detach=True)
        sec = parse_blob(blob)[0]
        memb = set(members.tolist())
        macset = set(macs.tolist())
        pred = {
            "nat_sessions": lambda k, v: _words(k[:, 0:4].copy()),
            "nat_reverse": lambda k, v: _words(v[:, 0:4].copy()),
            "eim_table": lambda k, v: _words(k[:, 0:4].copy()),
            "subscriber_nat": lambda k, v: _words(k), "qos_ingress": lambda k, v: _words(k),
            "qos_egress": lambda k, v: _words(k),
        }
        for m in TABLES:
            k, v = before[m]
            if m in pred:
                sel = np.isin(pred[m](k, v), list(memb)) if len(k) else np.zeros(0, bool)
            else:
                sel = np.isin(k.copy().view("<u8").reshape(-1), list(macset)) if len(k) else np.zeros(0, bool)
            assert _rows(m, *sec[m]) == _rows(m, k[sel], v[sel]), f"{m}: the export is not the predicate's selection"
            assert _rows(m, *dp.dump(m)) == _rows(m, k[~sel], v[~sel]), f"{m}: the detach removed something else"
        assert bytes(stale_k) in {bytes(r) for r in sec["nat_reverse"][0]}
        assert bytes(odd_k) not in {bytes(r) for r in sec["nat_sessions"][0]}
        assert set(_words(sec["li_targets"][0]).tolist()) == {int(ips[5])} & memb | ({int(ips[1])} & memb)
    finally:
        dp.close()


def test_consecutive_exports_select_their_own_sets():
    """Back-to-back exports of different sets, the first on a fresh context: each selects by its own addresses and
    MACs, never by the previous call's."""
    from bng_b200 import Dataplane
    dp, wl, ips = _small()
    fresh = Dataplane(**SMALL)
    try:
        k, v = dp.dump("nat_sessions")
        src = _words(k[:, 0:4].copy())
        bk, bv = dp.dump("subscriber_bindings")
        macs_all = S.sub_mac_key(np.arange(len(ips)))
        for j in range(7):
            sel_a, sel_m = ips[j::7], macs_all[(j + 3) % 7::7]
            sec = parse_blob(dp.sub_export(sel_a, sel_m))[0]
            want = np.isin(src, sel_a)
            assert _rows("nat_sessions", *sec["nat_sessions"]) == _rows("nat_sessions", k[want], v[want]), j
            wm = np.isin(bk.copy().view("<u8").reshape(-1), sel_m)
            assert _rows("subscriber_bindings", *sec["subscriber_bindings"]) == _rows("subscriber_bindings", bk[wm], bv[wm]), j
        blob = fresh.sub_export(ips[:5], macs_all[:5], detach=True)
        assert all(len(s[0]) == 0 for s in parse_blob(blob)[0].values())
    finally:
        dp.close()
        fresh.close()


def test_enospc_writes_and_removes_nothing():
    import ctypes as C
    dp, wl, ips = _small()
    try:
        addrs = ips[::3]
        before = _state(dp)
        need = C.c_uint64(0)
        assert dp.lib.bng_sub_export(dp.h, addrs.ctypes.data, len(addrs), None, 0, 1, None, 0, C.byref(need)) == -ENOSPC
        buf = np.full(need.value, 0xAB, np.uint8)
        n = C.c_uint64(0)
        assert dp.lib.bng_sub_export(dp.h, addrs.ctypes.data, len(addrs), None, 0, 1, buf.ctypes.data, need.value - 1,
                                     C.byref(n)) == -ENOSPC
        assert n.value == need.value and (buf == 0xAB).all()
        assert _state(dp) == before
        assert dp.lib.bng_sub_export(dp.h, addrs.ctypes.data, len(addrs), None, 0, 1, buf.ctypes.data, need.value,
                                     C.byref(n)) == 0
        assert n.value == need.value and _state(dp) != before
        assert dp.sub_import(buf.tobytes()) == 0 and _state(dp) == before
        # argument errors
        assert dp.lib.bng_sub_export(dp.h, None, 1, None, 0, 0, None, 0, C.byref(n)) == -EINVAL
        assert dp.lib.bng_sub_export(dp.h, None, 0, None, 1, 0, None, 0, C.byref(n)) == -EINVAL
        assert dp.lib.bng_sub_export(dp.h, None, 0, None, 0, 2, None, 0, C.byref(n)) == -EINVAL
        assert dp.lib.bng_sub_export(dp.h, None, 0, None, 0, 0, None, 0, None) == -EINVAL
    finally:
        dp.close()


def test_e2big_rollback_and_malformed_blobs():
    from bng_b200 import Dataplane
    dp, wl, ips = _small()
    tiny = Dataplane(max_batch=1 << 10, max_subscribers=1 << 10, max_nat_sessions=64, max_eim_mappings=64)
    try:
        before = _state(dp)
        tiny_before = _state(tiny)
        blob = dp.sub_export(ips[::2], S.sub_mac_key(np.arange(len(ips))[::2]), detach=True)
        r = tiny.lib.bng_sub_import(tiny.h, blob, len(blob))
        assert r == -E2BIG and _state(tiny) == tiny_before
        assert dp.sub_import(blob) == 0 and _state(dp) == before, "the rollback did not restore the source"
        # malformed blobs: nothing changes
        small = dp.sub_export(ips[:3], S.sub_mac_key(np.arange(3)))
        _, starts = parse_blob(small)
        bad = [b"BNGSNAP2" + small[8:]] + [small[:b] for b in starts] + [small[:-1], small + b"\0"]
        wrong_ks = bytearray(small)
        wrong_ks[starts[0] + 44:starts[0] + 48] = (8).to_bytes(4, "little")  # key_size of subscriber_nat
        bad.append(bytes(wrong_ks))
        for i, b in enumerate(bad):
            assert tiny.lib.bng_sub_import(tiny.h, b, len(b)) == -EINVAL, f"malformed blob {i} was taken"
        assert _state(tiny) == tiny_before
    finally:
        dp.close()
        tiny.close()


def test_no_per_batch_cost():
    from bng_b200 import Dataplane
    dp, wl, ips = _small()
    other = Dataplane(**SMALL)
    try:
        def launches(c):
            n0 = c.launch_count
            c.run("pipeline_up", wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0 + 5 * NS, stride=64)
            return c.launch_count - n0
        a0, b0 = launches(dp), launches(other)
        blob = dp.sub_export(ips[::2], S.sub_mac_key(np.arange(len(ips))[::2]), detach=True)
        assert other.sub_import(blob) == 0
        assert launches(dp) == a0 and launches(other) == b0
    finally:
        dp.close()
        other.close()


def test_delta_replication_across_a_move():
    from bng_b200 import Dataplane
    dp, wl, ips = _small()
    other = Dataplane(**SMALL)
    standby = [Dataplane(**SMALL), Dataplane(**SMALL)]
    try:
        other.acct_enable("pipeline_up")
        other.idle_enable("pipeline_up")
        act = [dp, other]
        for a, s in zip(act, standby):
            a.delta_enable()
            assert s.delta_apply(a.delta_export(exact=True)) == 0
        blob = dp.sub_export(ips[::3], S.sub_mac_key(np.arange(len(ips))[::3]), detach=True)
        assert other.sub_import(blob) == 0
        for a, s in zip(act, standby):
            assert s.delta_apply(a.delta_export(exact=True)) == 0
            for m in TABLES:
                assert _rows(m, *s.dump(m)) == _rows(m, *a.dump(m)), f"{m}: the standby differs from its active"
            sa, ra = s.acct_dump(), a.acct_dump()
            assert np.array_equal(sa[0], ra[0]) and np.array_equal(sa[1], ra[1])
    finally:
        for c in [dp, other] + standby:
            c.close()
