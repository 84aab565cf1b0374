"""NAT flow-state flush of a set of subscriber addresses (bng_nat_flush, include/bng_b200.h).

The reference has no such operation (its DeallocateNAT deletes the subscriber_nat entry only), so the semantics are
this repository's.  `flush_spec` restates them on top of the CPU oracle's plain map commands (dump / lookup / update /
delete, nothing else), and the device flush must leave exactly the same maps, counters and NAT_LOG_SESSION_DELETE
records, and the programs must go on computing what the oracle computes afterwards."""
import ctypes

import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import layouts as L
from bng_b200 import synth as S
from bng_b200 import workloads as W
from bng_b200.layouts import as_bytes

pytestmark = pytest.mark.gpu
NS = 10**9
MAPS = ("nat_sessions", "nat_reverse", "eim_table", "subscriber_nat")
ACTIVE = L.subscriber_nat.fields["sessions_active"][1]  # value offset of sessions_active


def _words(b):
    """u8[n, >=4] -> u32[n] of the first 4 bytes (addresses as the key words hold them)."""
    return np.ascontiguousarray(b[:, :4]).view("<u4").reshape(-1)


def flush_spec(o, addrs, now):
    """The flush through bpf(2)-style map commands on the oracle.  Returns ((sessions, reverse, eim) removed, the
    expected NAT_LOG_SESSION_DELETE records ordered by their bytes after the timestamp)."""
    a = set(int(x) for x in np.asarray(addrs, dtype="<u4").reshape(-1))
    k, v = o.dump("nat_sessions")
    logs = []
    if len(k):
        for kraw, s in zip(k[np.isin(_words(k), list(a))], v[np.isin(_words(k), list(a))].view(L.nat_session).reshape(-1)):
            assert o.delete("nat_sessions", kraw) == 0
            sv = o.lookup("subscriber_nat", np.ascontiguousarray(s["orig_ip"]))
            rec = np.zeros(1, L.nat_log_entry)
            rec["timestamp"], rec["event_type"] = now, 2
            rec["subscriber_id"] = 0 if sv is None else int(sv.view(L.subscriber_nat)["block"]["subscriber_id"][0])
            rec["private_ip"], rec["public_ip"] = s["orig_ip"], s["nat_ip"]
            rec["private_port"], rec["public_port"] = s["orig_port"], s["nat_port"]
            rec["dest_ip"], rec["dest_port"], rec["protocol"] = s["dest_ip"], s["dest_port"], s["protocol"]
            logs.append(bytes(as_bytes(rec)[0]))
    n_ses = len(logs)
    counts = [n_ses]
    for m, col in (("nat_reverse", "v"), ("eim_table", "k")):
        k, v = o.dump(m)
        hit = np.isin(_words(v if col == "v" else k), list(a)) if len(k) else np.zeros(0, bool)
        for kraw in k[hit]:
            assert o.delete(m, kraw) == 0
        counts.append(int(hit.sum()))
    for x in sorted(a):
        kb = np.array([x], "<u4").view(np.uint8)
        sv = o.lookup("subscriber_nat", kb)
        if sv is not None:
            sn = np.array(sv, np.uint8).copy()
            sn[ACTIVE:ACTIVE + 8] = 0
            assert o.update_batch("subscriber_nat", kb.reshape(1, 4), sn.reshape(1, -1), 2) == 0
    logs.sort(key=lambda r: r[8:])
    recs = np.frombuffer(b"".join(logs), np.uint8).reshape(-1, 40) if logs else np.zeros((0, 40), np.uint8)
    return tuple(counts), recs


def expect_from_dumps(dumps, addrs):
    """What a flush of addrs leaves, computed from dumps {map: (keys, values)} taken before it: (tables, counts)."""
    a = np.asarray(addrs, dtype="<u4").reshape(-1)
    out, counts = {}, []
    for m, col in (("nat_sessions", 0), ("nat_reverse", 1), ("eim_table", 0)):
        k, v = dumps[m]
        hit = np.isin(_words((k, v)[col]), a) if len(k) else np.zeros(0, bool)
        out[m] = (k[~hit], v[~hit])
        counts.append(int(hit.sum()))
    k, v = dumps["subscriber_nat"]
    v = v.copy()
    v[np.isin(_words(k), a), ACTIVE:ACTIVE + 8] = 0
    out["subscriber_nat"] = (k, v)
    return out, tuple(counts)


def _state(be):
    out = {}
    for m in MAPS:
        k, v = be.dump(m)
        out["k_" + m], out["v_" + m] = k, harness.mask_padding(m, v) if len(v) else v
    out["stats"] = be.stats("nat_stats_map")
    return out


def _masked_logs(r):
    return harness.mask_padding("nat_log_rb", r) if len(r) else r.reshape(0, 40)


def _assert_same(ora, gpu, what):
    a, b = _state(ora), _state(gpu)
    for key in a:
        assert np.array_equal(a[key], b[key]), f"{what}: {key} differs"


def _flush_sets(ora):
    """One subscriber, a third of them with a duplicate and 0 / 0xFFFFFFFF, an address with no state, the rest."""
    subs = _words(ora.dump("subscriber_nat")[0])
    third = subs[1::3]
    return [subs[:1], np.concatenate([third, third[:2], np.array([0, 0xFFFFFFFF], "<u4")]),
            np.array([0x04030201], "<u4"), subs]


SCRIPTS = {
    "nat_eim": lambda: scenarios.nat_script(seed=0xF1A5, flags=0x0F, n_subs=24, pps=64, n=2500, name="nat_flush"),
    "nat_noeim": lambda: scenarios.nat_script(seed=0xF1A6, flags=0x0E, n_subs=24, pps=64, n=2500, name="nat_flush_noeim"),
    "pipeline_up": lambda: scenarios.pipeline_script(seed=0xF1A7),
    "pipeline_tc": lambda: scenarios.pipeline_script(seed=0xF1A8, prog="pipeline_tc"),
}


def _require_oracle(ora_kind):
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")


@pytest.mark.parametrize("name", list(SCRIPTS))
def test_flush_matches_the_spec_on_the_oracle(name, ora_kind):
    _require_oracle(ora_kind)
    sc = SCRIPTS[name]()
    ora, gpu = harness.OracleBackend(ora_kind), harness.GpuBackend()
    try:
        harness.compare(harness.run_script(ora, sc), harness.run_script(gpu, sc), f"{name}: state before the flush")
        stats0 = gpu.stats("nat_stats_map").copy()
        assert gpu.dp.map_info("nat_sessions")["count"] > 0
        for i, addrs in enumerate(_flush_sets(ora)):
            now = (100 + 10 * i) * NS
            want, want_logs = flush_spec(ora.o, addrs, now)
            got = gpu.dp.nat_flush(addrs, now)
            assert got == want, f"flush {i}: removed {got}, spec says {want}"
            got_logs = gpu.dp.drain("nat_log_rb")
            assert np.array_equal(_masked_logs(got_logs), _masked_logs(want_logs)), f"flush {i}: records differ"
            _assert_same(ora, gpu, f"{name}, flush {i}")
        assert np.array_equal(gpu.stats("nat_stats_map"), stats0), "nat_stats changed"
        for m in ("nat_sessions", "nat_reverse", "eim_table"):
            assert gpu.dp.map_info(m)["count"] == 0, m  # every subscriber has been flushed by now
        assert gpu.dp.lru_overflow == 0
    finally:
        gpu.close()
        ora.close()


def _device_run_then_flush(dp, prog, arena, lens, now, off16, stride, prio, addrs, fnow):
    """A device-resident batch with the flush queued right behind it: no host synchronisation in between."""
    import torch
    from bng_b200 import MEM_DEVICE
    dev = torch.device("cuda")
    ta = torch.from_numpy(arena.copy()).to(dev)
    tl = torch.from_numpy(lens.view(np.int32).copy()).to(dev)
    to = None if off16 is None else torch.from_numpy(off16.view(np.int32).copy()).to(dev)
    tp = None if prio is None else torch.from_numpy(prio.view(np.int32).copy()).to(dev)
    tv = torch.zeros(len(lens), dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()  # the library's stream does not wait for torch's
    dp.run(prog, ta, tl, now, off16=to, stride=stride, priority=tp, verdict=tv, mem=MEM_DEVICE, arena_bytes=arena.nbytes)
    counts = dp.nat_flush(addrs, fnow)
    torch.cuda.synchronize()
    arena[:] = ta.cpu().numpy()
    lens[:] = tl.cpu().numpy().view(np.uint32)
    if prio is not None:
        prio[:] = tp.cpu().numpy().view(np.uint32)
    return tv.cpu().numpy(), counts


@pytest.mark.parametrize("feed", [False, True, "device"], ids=["pageable", "pinned", "device"])
@pytest.mark.parametrize("name", ["nat_eim", "pipeline_tc"])
def test_traffic_after_the_flush(name, feed, ora_kind):
    """The script's batches again, each followed by a flush of another set: the frames of the flushed subscribers
    create new state, and everything stays bit-identical to the oracle with the spec's deletions."""
    _require_oracle(ora_kind)
    sc = SCRIPTS[name]()
    ora, gpu = harness.OracleBackend(ora_kind), harness.GpuBackend(pinned=feed)
    try:
        harness.compare(harness.run_script(ora, sc), harness.run_script(gpu, sc), f"{name}/{feed}: before")
        sets = _flush_sets(ora)
        runs = [st for st in sc.steps if st[0] == "run"]
        for j, (_, prog, arena, lens, now, off16, stride, prio, _nv) in enumerate(runs):
            now += 1000 * NS
            addrs = sets[j % len(sets)]
            ao, lo, po = arena.copy(), lens.copy(), None if prio is None else prio.copy()
            vo = ora.run(prog, ao, lo, now, off16, stride, po)
            want_run_logs = ora.drain("nat_log_rb")
            want, want_logs = flush_spec(ora.o, addrs, now + NS)
            ag, lg, pg = arena.copy(), lens.copy(), None if prio is None else prio.copy()
            if feed == "device":
                vg, got = _device_run_then_flush(gpu.dp, prog, ag, lg, now, off16, stride, pg, addrs, now + NS)
            else:
                vg = gpu.run(prog, ag, lg, now, off16, stride, pg)
                got = gpu.dp.nat_flush(addrs, now + NS)
            what = f"{name}/{feed}, batch {j}"
            assert np.array_equal(np.asarray(vg), np.asarray(vo)), f"{what}: verdicts differ"
            assert np.array_equal(ag, ao) and np.array_equal(lg, lo), f"{what}: frames differ"
            assert got == want, f"{what}: removed {got}, spec says {want}"
            both = [r for r in (want_run_logs, want_logs) if len(r)]
            want_all = np.concatenate(both, axis=0) if both else np.zeros((0, 40), np.uint8)
            assert np.array_equal(_masked_logs(gpu.drain("nat_log_rb")), _masked_logs(want_all)), f"{what}: records differ"
            sg, so = gpu.drain("spoof_events"), ora.drain("spoof_events")
            assert (len(sg) == len(so) == 0) or np.array_equal(harness.mask_padding("spoof_events", sg),
                                                               harness.mask_padding("spoof_events", so)), \
                f"{what}: spoof events differ"
            _assert_same(ora, gpu, what)
        assert gpu.dp.lru_overflow == 0 and gpu.dp.events_lost == 0
    finally:
        gpu.close()
        ora.close()


def _frames(sub, sport, lens):
    return S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), np.uint32(0x08080808), 17,
                          sport, 53, lens, l4_check=0x3333)


def _replies(out):
    rep = out.copy()
    rep[:, 26:30], rep[:, 30:34] = out[:, 30:34], out[:, 26:30]
    rep[:, 34:36], rep[:, 36:38] = out[:, 36:38], out[:, 34:36]
    return rep


@pytest.mark.parametrize("flush", [True, False], ids=["flushed", "inherited"])
def test_successor_of_an_address(flush, ora_kind):
    """Subscriber X leaves and its address comes back with another subscriber's freed block.  Flushed, its next
    frames translate into the new block and replies to the old public ports pass untranslated.  Without the flush
    (the reference's behaviour, which this feature exists for) both the oracle and the GPU keep the old translation
    and DNAT the old ports to the address's new holder."""
    _require_oracle(ora_kind)
    ora, gpu = harness.OracleBackend(ora_kind), harness.GpuBackend()
    try:
        sc = harness.Script("maps")
        scenarios.nat_maps(sc, 4, 64, 0x0F)
        for st in sc.steps:
            assert ora.update(*st[1:5]) == 0 and gpu.update(*st[1:5]) == 0
        sub_keys, sub_vals = gpu.dump("subscriber_nat")
        x_key = S.ip_bytes(S.sub_ip(np.array([0])))[0]
        y_key = S.ip_bytes(S.sub_ip(np.array([1])))[0]
        y_val = sub_vals[np.all(sub_keys == y_key, axis=1)][0]
        sub = np.zeros(6, np.int64)
        lens = np.full(6, 64, np.uint32)
        up = _frames(sub, np.arange(30000, 30006, dtype=np.uint32), lens)

        def run(prog, frames, now):
            ao, ag = frames.reshape(-1).copy(), frames.reshape(-1).copy()
            vo = ora.run(prog, ao, lens.copy(), now, None, 64, None)
            vg = gpu.run(prog, ag, lens.copy(), now, None, 64, None)
            assert np.array_equal(np.asarray(vo), np.asarray(vg)) and np.array_equal(ao, ag), f"{prog} at {now}: differs"
            return ag.reshape(-1, 64)

        first = run("nat44_egress", up, 1 * NS)
        assert (first[:, 26:30] != up[:, 26:30]).any(axis=1).all()
        for key in (x_key, y_key):  # X leaves; Y leaves too, freeing its block
            if flush:
                want, _ = flush_spec(ora.o, key.view("<u4"), 2 * NS)
                assert gpu.dp.nat_flush(key.view("<u4"), 2 * NS) == want
            assert ora.delete("subscriber_nat", key) == 0 and gpu.delete("subscriber_nat", key) == 0
        assert ora.update("subscriber_nat", x_key.reshape(1, 4), y_val.reshape(1, -1), 0) == 0
        assert gpu.update("subscriber_nat", x_key.reshape(1, 4), y_val.reshape(1, -1), 0) == 0
        again = run("nat44_egress", up, 3 * NS)
        y_blk = y_val.view(L.subscriber_nat)["block"][0]
        ports = again[:, 34].astype(np.uint32) << 8 | again[:, 35]
        back = run("nat44_ingress", _replies(first), 4 * NS)
        if flush:
            assert (again[:, 26:30] == np.asarray(y_blk["public_ip"])).all()
            assert ((ports >= int(y_blk["port_start"])) & (ports <= int(y_blk["port_end"]))).all(), ports
            assert np.array_equal(back, _replies(first)), "replies to the old ports were translated"
        else:
            assert np.array_equal(again, first), "the old sessions were not inherited"
            assert (back[:, 30:34] == up[:, 26:30]).all(), "replies to the old ports did not reach the new holder"
        _assert_same(ora, gpu, f"successor ({'flushed' if flush else 'inherited'})")
    finally:
        gpu.close()
        ora.close()


def _dumps(dp):
    return {m: dp.dump(m) for m in MAPS}


def _assert_tables(dp, want, what):
    for m in MAPS:
        k, v = dp.dump(m)
        wk, wv = want[m]
        assert np.array_equal(k, wk), f"{what}: {m} keys differ"
        assert np.array_equal(harness.mask_padding(m, v) if len(v) else v, harness.mask_padding(m, wv) if len(wv) else wv), \
            f"{what}: {m} values differ"


def test_flush_at_the_reference_capacities():
    """2^20 frames of pipeline_imix into tables of the reference's sizes (4 M sessions, 2 M EIM mappings), then a
    flush of 1 000 subscriber addresses: the tables are the pre-flush dumps minus what the predicates select."""
    from bng_b200 import Dataplane
    n = 1 << 20
    wl = W.build("pipeline_imix", n)
    dp = Dataplane(max_batch=n)
    try:
        for m, k, v in wl.maps:
            assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
        for prog, h, l in wl.prewarm:
            dp.run(prog, h.reshape(-1).copy(), l.copy(), wl.now0 - 1, stride=64)
        dp.run(wl.prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0, stride=64)
        dp.drain("nat_log_rb")
        before = _dumps(dp)
        addrs = _words(before["subscriber_nat"][0])[::7][:1000]
        assert len(addrs) == 1000
        want, counts = expect_from_dumps(before, addrs)
        got = dp.nat_flush(addrs, wl.now0 + NS)
        assert got == counts and counts[0] > 0 and counts[1] > 0 and counts[2] > 0, (got, counts)
        ring = (dp.map_info("nat_log_rb")["max_entries"] - 1) // 48  # records of 8 + 40 bytes the kernel's ring holds
        assert len(dp.drain("nat_log_rb")) == min(counts[0], ring)
        _assert_tables(dp, want, "2^20 frames, 1 000 addresses")
        assert dp.lru_overflow == 0
    finally:
        dp.close()


def test_flush_that_tombstones_a_quarter_rebuilds_the_flow_tables():
    from bng_b200 import Dataplane
    dp = Dataplane(max_subscribers=1 << 10, max_nat_sessions=256, max_eim_mappings=256, max_batch=1 << 12)
    try:
        sc = harness.Script("maps")
        n_subs = 20
        scenarios.nat_maps(sc, n_subs, 1024, 0x0F)
        for st in sc.steps:
            assert dp.update_batch(st[1], st[2], st[3], st[4]) == 0
        sub = np.repeat(np.arange(n_subs), 8)
        lens = np.full(len(sub), 64, np.uint32)
        h = _frames(sub, (3000 + np.tile(np.arange(8), n_subs)).astype(np.uint32), lens)
        dp.run("nat44_egress", h.reshape(-1).copy(), lens, 10 * NS, stride=64)
        assert dp.map_info("nat_sessions")["count"] == 160  # of 512 slots: 160 tombstones are more than a quarter
        subs = _words(dp.dump("subscriber_nat")[0])
        r0 = dp.table_rebuilds
        before = _dumps(dp)
        want, counts = expect_from_dumps(before, subs[:1])
        assert dp.nat_flush(subs[:1], 11 * NS) == counts == (8, 8, 8)
        assert dp.table_rebuilds == r0, "8 tombstones of 512 slots rebuilt the tables"
        _assert_tables(dp, want, "one subscriber")
        before = _dumps(dp)
        want, counts = expect_from_dumps(before, subs[1:])
        assert dp.nat_flush(subs[1:], 12 * NS) == counts == (152, 152, 152)
        assert dp.table_rebuilds > r0, "160 tombstones of 512 slots did not rebuild the tables"
        _assert_tables(dp, want, "after the rebuild")
        # the rebuilt tables work: the same flows are created again
        dp.run("nat44_egress", h.reshape(-1).copy(), lens, 13 * NS, stride=64)
        assert dp.map_info("nat_sessions")["count"] == 160 and dp.lru_overflow == 0
    finally:
        dp.close()


def test_accounting_records_and_errors():
    from bng_b200 import Dataplane
    from bng_b200.dataplane import load_library
    dp = Dataplane(max_subscribers=1 << 10, max_nat_sessions=1 << 10, max_eim_mappings=1 << 10, max_batch=1 << 12)
    try:
        sc = harness.Script("maps")
        scenarios.nat_maps(sc, 8, 64, 0x0F)
        for st in sc.steps:
            assert dp.update_batch(st[1], st[2], st[3], st[4]) == 0
        dp.acct_enable("nat44_egress")
        sub = np.repeat(np.arange(8), 3)
        lens = np.full(len(sub), 64, np.uint32)
        dp.run("nat44_egress", _frames(sub, (4000 + np.tile(np.arange(3), 8)).astype(np.uint32), lens).reshape(-1).copy(),
               lens, 5 * NS, stride=64)
        subs = _words(dp.dump("subscriber_nat")[0])
        rec0, found0 = dp.acct_read(subs)
        assert found0.all() and (rec0["up_packets"] == 3).all()
        assert dp.nat_flush(subs[:3], 6 * NS) == (9, 9, 9)
        rec1, found1 = dp.acct_read(subs)
        assert found1.all() and np.array_equal(rec0, rec1), "a flush changed accounting records"
        # n == 0: staged upserts are applied, nothing is removed
        k, v = dp.dump("subscriber_nat")
        nv = v[3].copy()
        nv[ACTIVE:ACTIVE + 8] = 7
        assert dp.update_staged("subscriber_nat", k[3], nv) == 0 and dp.staged_info()["pending"] == 1
        seq = dp.map_info("nat_sessions")["count"]
        assert dp.nat_flush(np.zeros(0, "<u4"), 7 * NS) == (0, 0, 0)
        assert dp.staged_info()["pending"] == 0 and dp.map_info("nat_sessions")["count"] == seq
        assert np.array_equal(dp.lookup("subscriber_nat", k[3]), nv)
        lib = load_library()
        out = (ctypes.c_uint64 * 3)(5, 5, 5)
        assert lib.bng_nat_flush(None, None, 0, 0, out) == -22
        assert lib.bng_nat_flush(dp.h, None, 1, 0, out) == -22
        assert lib.bng_nat_flush(dp.h, None, 0, 8 * NS, out) == 0 and list(out) == [0, 0, 0]
        assert lib.bng_nat_flush(dp.h, subs.ctypes.data, 1, 8 * NS, None) == 0  # counts are optional
    finally:
        dp.close()


@pytest.mark.parametrize("world", [2, 8])
def test_flush_on_owner_shards_equals_the_unsharded_flush(world):
    from bng_b200 import Dataplane
    n, n_subs = 1 << 16, 1_000
    wl = W.pipeline(n, 0, 1, n_subs=n_subs, flows_per_sub=16, imix=False)
    sub = np.arange(n_subs, dtype=np.uint32)
    ip_keys = S.ip_bytes(S.sub_ip(sub))
    ip_shard = dict(zip(_words(ip_keys).tolist(), S.shard_of_mac(S.sub_mac_key(sub), world).tolist()))
    flush = np.concatenate([_words(ip_keys)[::3], np.array([0x04030201], "<u4")])  # a third, and one nobody owns
    mac_of = lambda h: sum(h[:, 6 + i].astype(np.uint64) << np.uint64(8 * (5 - i)) for i in range(6))

    def run(dp, rank):
        for m, k, v in wl.maps:
            kb, vb = as_bytes(k), as_bytes(v)
            if rank is not None and m == "subscriber_bindings":
                keep = S.shard_of_mac(k.astype(np.uint64), world) == rank
                kb, vb = kb[keep], vb[keep]
            elif rank is not None and m in ("qos_ingress", "subscriber_nat"):
                keep = np.array([ip_shard[int(x)] == rank for x in _words(kb)])
                kb, vb = kb[keep], vb[keep]
            assert dp.update_batch(m, kb, vb) == 0, m
        for prog, h, l in wl.prewarm:
            mine = np.ones(len(h), bool) if rank is None else S.shard_of_mac(mac_of(h), world) == rank
            dp.run(prog, h[mine].reshape(-1).copy(), l[mine].copy(), wl.now0 - 1, stride=64)
        mine = np.ones(n, bool) if rank is None else S.shard_of_mac(mac_of(wl.headers), world) == rank
        dp.run(wl.prog, wl.headers[mine].reshape(-1).copy(), wl.lens[mine].copy(), wl.now0, stride=64)
        owned = flush if rank is None else np.array([a for a in flush if ip_shard.get(int(a), rank) == rank], "<u4")
        counts = dp.nat_flush(owned, wl.now0 + NS)
        return counts, _dumps(dp)

    opts = dict(max_batch=n, max_subscribers=4 * n_subs, max_nat_sessions=1 << 17, max_eim_mappings=1 << 17)
    dp = Dataplane(**opts)
    try:
        want_counts, want = run(dp, None)
    finally:
        dp.close()
    assert want_counts[0] > 0
    got_counts, parts = np.zeros(3, np.int64), {m: [] for m in MAPS}
    for rank in range(world):
        dp = Dataplane(rank=rank, world=world, **opts)
        try:
            c, d = run(dp, rank)
            assert dp.lru_overflow == 0
        finally:
            dp.close()
        got_counts += c
        for m in MAPS:
            parts[m].append(np.concatenate([d[m][0], harness.mask_padding(m, d[m][1])], axis=1))
    assert tuple(got_counts.tolist()) == want_counts
    for m in MAPS:
        k, v = want[m]
        rows = sorted(bytes(r) for r in np.concatenate([k, harness.mask_padding(m, v)], axis=1))
        assert sorted(bytes(r) for p in parts[m] for r in p) == rows, f"{m}: union of the shards differs"
