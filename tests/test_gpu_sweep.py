"""Session expiry sweep and LRU behaviour of the NAT flow tables (SURVEY.md §8f-3).

The reference declares the timeouts (bpf/nat44.c:50-53) and enforces them nowhere (pkg/nat/manager.go:667-679 only
logs), so the sweep's semantics are this repository's (include/bng_b200.h, bng_sweep).  `sweep_spec` below restates
them on top of the CPU oracle's plain map commands — lookup / update / delete, nothing else — and the device sweep
must leave exactly the same maps, counters and NAT_LOG_SESSION_DELETE records."""
import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import layouts as L
from bng_b200 import synth as S

pytestmark = pytest.mark.gpu
NS = 10**9


def timeout_ns(proto, state):
    if proto == 1:
        return 60 * NS
    if proto == 6:
        return 7200 * NS if state == 1 else 240 * NS
    return 120 * NS


def sweep_spec(o, now):
    """The sweep, one session at a time, through bpf(2)-style map commands on the oracle.  Returns the expected
    NAT_LOG_SESSION_DELETE records (ordered by their bytes after the timestamp)."""
    k, v = o.dump("nat_sessions")
    keys, ses = k.view(L.nat_key).reshape(-1), v.view(L.nat_session).reshape(-1)
    logs = []
    for kraw, key, s in zip(k, keys, ses):
        if now < int(s["last_seen"]) or now - int(s["last_seen"]) <= timeout_ns(int(s["protocol"]), int(s["state"])):
            continue
        assert o.delete("nat_sessions", kraw) == 0
        rk = np.zeros(1, L.nat_key)
        rk["src_ip"], rk["dst_ip"] = s["dest_ip"], s["nat_ip"]
        rk["src_port"], rk["dst_port"], rk["protocol"] = s["dest_port"], s["nat_port"], s["protocol"]
        rkb = L.as_bytes(rk)[0]
        rv = o.lookup("nat_reverse", rkb)
        if rv is not None and bytes(rv) == bytes(kraw):
            assert o.delete("nat_reverse", rkb) == 0
        ek = np.zeros(1, L.eim_key)
        ek["internal_ip"], ek["protocol"] = s["orig_ip"], s["protocol"]
        ek["internal_port"] = int(s["orig_port"][0]) | (int(s["orig_port"][1]) << 8)
        ekb = L.as_bytes(ek)[0]
        m = o.lookup("eim_table", ekb)
        if m is not None:
            mm = m.view(L.eim_mapping).copy()
            if int(mm["ref_count"][0]) == 1:
                assert o.delete("eim_table", ekb) == 0
            elif int(mm["ref_count"][0]) > 1:
                mm["ref_count"] -= 1
                assert o.update_batch("eim_table", L.as_bytes(ek), L.as_bytes(mm), 2) == 0
        sub_id = 0
        sv = o.lookup("subscriber_nat", np.ascontiguousarray(s["orig_ip"]))
        if sv is not None:
            sn = sv.view(L.subscriber_nat).copy()
            sub_id = int(sn["block"]["subscriber_id"][0])
            if int(sn["sessions_active"][0]) > 0:
                sn["sessions_active"] -= 1
                assert o.update_batch("subscriber_nat", s["orig_ip"].reshape(1, 4), L.as_bytes(sn), 2) == 0
        st = o.lookup("nat_stats_map", np.zeros(4, np.uint8)).view(L.nat_stats).copy()
        st["sessions_expired"] += 1
        assert o.update_batch("nat_stats_map", np.zeros((1, 4), np.uint8), L.as_bytes(st)) == 0
        rec = np.zeros(1, L.nat_log_entry)
        rec["timestamp"], rec["event_type"], rec["subscriber_id"] = now, 2, sub_id
        rec["private_ip"], rec["public_ip"] = s["orig_ip"], s["nat_ip"]
        rec["private_port"], rec["public_port"] = s["orig_port"], s["nat_port"]
        rec["dest_ip"], rec["dest_port"], rec["protocol"] = s["dest_ip"], s["dest_port"], s["protocol"]
        logs.append(bytes(L.as_bytes(rec)[0]))
    logs.sort(key=lambda r: r[8:])
    return np.frombuffer(b"".join(logs), np.uint8).reshape(-1, 40) if logs else np.zeros((0, 40), np.uint8)


MAPS = ("nat_sessions", "nat_reverse", "eim_table", "subscriber_nat")


def _state(be):
    out = {}
    for m in MAPS:
        k, v = be.dump(m)
        out["k_" + m], out["v_" + m] = k, harness.mask_padding(m, v) if len(v) else v
    out["stats"] = be.stats("nat_stats_map")
    return out


@pytest.mark.parametrize("flags", [0x0F, 0x0E], ids=["eim", "noeim"])
def test_sweep_matches_the_spec_on_the_oracle(flags, ora_kind):
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    # the nat scenario: three egress batches a second apart (t = 5, 6, 7 s), return traffic that moves TCP
    # sessions to ESTABLISHED / CLOSING — then sweeps at times that cross each timeout class
    sc = scenarios.nat_script(seed=0x5EE9, flags=flags, n_subs=24, pps=64, n=2500, name="nat_sweep")
    ora, gpu = harness.OracleBackend(ora_kind), harness.GpuBackend()
    try:
        ro, rg = harness.run_script(ora, sc), harness.run_script(gpu, sc)
        harness.compare(ro, rg, "state before the sweep")
        total = 0
        for now in (9 * NS, 66 * NS, 68 * NS, 127 * NS, 130 * NS, 250 * NS, 7000 * NS, 7300 * NS, 8000 * NS):
            want_logs = sweep_spec(ora.o, now)
            n = gpu.dp.sweep(now)
            got_logs = gpu.dp.drain("nat_log_rb")
            assert n == len(want_logs), f"sweep at {now // NS} s: {n} sessions removed, spec says {len(want_logs)}"
            assert np.array_equal(harness.mask_padding("nat_log_rb", got_logs) if len(got_logs) else got_logs.reshape(0, 40),
                                  harness.mask_padding("nat_log_rb", want_logs) if len(want_logs) else want_logs), \
                f"sweep at {now // NS} s: SESSION_DELETE records differ"
            a, b = _state(ora), _state(gpu)
            for key in a:
                assert np.array_equal(a[key], b[key]), f"sweep at {now // NS} s: {key} differs"
            total += n
        assert total == len(ro["tk_nat_sessions"]) and gpu.dp.map_info("nat_sessions")["count"] == 0
        assert gpu.dp.map_info("nat_reverse")["count"] == len(ora.dump("nat_reverse")[0])
        if flags & 1:
            assert gpu.dp.map_info("eim_table")["count"] == 0  # every mapping went with its last session
        assert gpu.dp.lru_overflow == 0
    finally:
        gpu.close()
        ora.close()


def test_full_lru_tables_evict_instead_of_failing():
    """nat_sessions / nat_reverse / eim_table are BPF_MAP_TYPE_LRU_HASH (bpf/nat44.c:218-244): an insert into a full
    map makes room.  200 subscribers x 8 new flows per batch into tables of 512 entries: nothing is ever refused,
    the tables stay at their size, what survives is recent, and replies to surviving flows are still translated.
    Every eviction leaves a tombstone, so the flow tables are rebuilt on the way."""
    _lru_churn("pageable")


def test_full_lru_tables_are_compacted_on_the_device_path():
    """The same churn with device-resident batches that nothing but torch ever synchronises: the flow tables must
    still be rebuilt (a table without EMPTY slots makes every lookup of an absent key walk all of it)."""
    _lru_churn("device")


def _lru_churn(feed):
    import torch
    from bng_b200 import MEM_DEVICE, Dataplane
    cap = 512
    dp = Dataplane(max_subscribers=1 << 10, max_nat_sessions=cap, max_eim_mappings=cap, max_batch=1 << 13)

    def run(prog, a, lens, now):
        if feed == "pageable":
            return np.asarray(dp.run(prog, a, lens, now, stride=64))
        ta, tl = torch.from_numpy(a).cuda(), torch.from_numpy(lens.view(np.int32)).cuda()
        tv = torch.zeros(len(lens), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        dp.run(prog, ta, tl, now, stride=64, verdict=tv, mem=MEM_DEVICE)
        torch.cuda.synchronize()
        a[:] = ta.cpu().numpy()
        return tv.cpu().numpy()

    try:
        sc = harness.Script("maps")
        n_subs = 200
        scenarios.nat_maps(sc, n_subs, 64, 0x0F)
        for st in sc.steps:
            assert dp.update_batch(st[1], st[2], st[3], st[4]) == 0
        last = None
        for b in range(12):
            sub = np.repeat(np.arange(n_subs), 8)
            sport = (1000 + 100 * b + np.tile(np.arange(8), n_subs)).astype(np.uint32)
            lens = np.full(len(sub), 64, np.uint32)
            h = S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), np.uint32(0x08080808), 17, sport, 53,
                               lens, l4_check=0x2222)
            a = h.reshape(-1).copy()
            v = run("nat44_egress", a, lens, (10 + b) * NS)
            assert (v == 0).all()
            assert (a.reshape(-1, 64)[:, 26:30] != h[:, 26:30]).any(axis=1).all(), "a frame left untranslated"
            last = a.reshape(-1, 64).copy()
            for m in ("nat_sessions", "nat_reverse", "eim_table"):
                assert dp.map_info(m)["count"] <= cap, m
        assert dp.lru_overflow == 0
        assert dp.lru_evictions >= 11 * n_subs * 8  # every batch after the first pushed something out
        assert dp.table_rebuilds >= 3, f"{dp.lru_evictions} evictions, {dp.table_rebuilds} rebuilds of the flow tables"
        k, v = dp.dump("nat_sessions")
        ses = v.view(L.nat_session).reshape(-1)
        assert len(ses) >= cap - 64 and int(ses["last_seen"].min()) >= 19 * NS, "old sessions survived newer ones"
        # replies to the newest flows: those whose session and reverse entry both survived are DNATed
        out = last.copy()
        out[:, 26:30], out[:, 30:34] = last[:, 30:34], last[:, 26:30]
        out[:, 34:36], out[:, 36:38] = last[:, 36:38], last[:, 34:36]
        before = dp.stats("nat_stats_map")[1]
        r = out.reshape(-1).copy()
        run("nat44_ingress", r, np.full(len(out), 64, np.uint32), 30 * NS)
        dnat = int(dp.stats("nat_stats_map")[1] - before)
        assert dnat >= cap // 8, f"only {dnat} replies translated"  # session AND reverse entry survived (independent evictions)
        back = r.reshape(-1, 64)
        hit = (back[:, 30:34] != out[:, 30:34]).any(axis=1)
        assert int(hit.sum()) == dnat
    finally:
        dp.close()


def test_session_churn_rebuilds_the_flow_tables():
    """Create / expire / create ...: tombstones pile up until bng_sweep rebuilds the three flow tables; traffic before and
    after the rebuild is translated the same way and the tables hold exactly the live flows."""
    from bng_b200 import Dataplane
    dp = Dataplane(max_subscribers=1 << 10, max_nat_sessions=256, max_eim_mappings=256, max_batch=1 << 12)
    try:
        sc = harness.Script("maps")
        n_subs = 20
        scenarios.nat_maps(sc, n_subs, 1024, 0x0F)
        for st in sc.steps:
            assert dp.update_batch(st[1], st[2], st[3], st[4]) == 0
        rebuilds = 0
        for rnd in range(8):
            sub = np.repeat(np.arange(n_subs), 5)
            sport = (2000 + 10 * rnd + np.tile(np.arange(5), n_subs)).astype(np.uint32)
            lens = np.full(len(sub), 64, np.uint32)
            h = S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), np.uint32(0x08080808), 17, sport, 53,
                               lens, l4_check=0x2222)
            t0 = (1000 * rnd + 10) * NS
            a = h.reshape(-1).copy()
            v = dp.run("nat44_egress", a, lens, t0, stride=64)
            assert (np.asarray(v) == 0).all() and (a.reshape(-1, 64)[:, 26:30] != h[:, 26:30]).any(axis=1).all()
            assert dp.map_info("nat_sessions")["count"] == 100 and dp.map_info("eim_table")["count"] == 100
            # the flows answer (DNAT works through whatever state the tables are in) ...
            out = a.reshape(-1, 64).copy()
            rep = out.copy()
            rep[:, 26:30], rep[:, 30:34] = out[:, 30:34], out[:, 26:30]
            rep[:, 34:36], rep[:, 36:38] = out[:, 36:38], out[:, 34:36]
            r = rep.reshape(-1).copy()
            dp.run("nat44_ingress", r, lens.copy(), t0 + NS, stride=64)
            assert (r.reshape(-1, 64)[:, 30:34] == h[:, 26:30]).all()
            # ... and all expire 200 s later
            assert dp.sweep(t0 + 200 * NS) == 100
            for m in ("nat_sessions", "nat_reverse", "eim_table"):
                assert dp.map_info(m)["count"] == 0, m
            rebuilds = dp.table_rebuilds
        assert rebuilds >= 3, "512-slot tables with 100 tombstones per round were never compacted"
        assert dp.lru_overflow == 0
    finally:
        dp.close()


EPOCH_PERIOD = 65535  # bng_prog_run: epoch = batch_seq % 65535 + 1; every epoch is cleared when it comes round to 1


def epoch_wrap_script():
    """A session hit stores last_seen only when the session's 16-bit epoch differs from the batch's (common.cuh,
    ses_touch), so the epochs are all cleared when the batch counter comes round to the same values again.  Two
    sets of flows, each split four ways: hits of nat44_egress, replies through nat44_ingress, pipeline_up,
    pipeline_tc (half the subscribers with a rate-limited bucket: TC runs NAT after it, in the ordered phase).
      set 2 is touched in the four batches before the reset (batch 65 535) and in the four from it on;
      set 1 is touched in batches 6-9 and then not again until batches 6-9 + 65 535, with the same epoch values.
    Everything between is 1-frame ARP batches of antispoof_ingress.  Returns (script, batches)."""
    n_subs, ns = 16, 10**9
    sc = harness.Script("epoch_wrap")
    keys, v = S.bindings(n_subs)
    sc.update("subscriber_bindings", keys, v)
    cfg = np.zeros(1, L.antispoof_config)
    cfg["default_mode"] = 1
    sc.update1("antispoof_config", np.uint32(0), cfg)
    scenarios.nat_maps(sc, n_subs, 64, 0x0F)
    qk, qv = S.qos_buckets(n_subs // 2)
    qv["rate_bps"], qv["burst_bytes"] = 10**12, 1 << 30
    qv["tokens"] = qv["burst_bytes"]
    sc.update("qos_ingress", qk, qv)
    sub = np.tile(np.arange(n_subs), 2)  # two frames of every flow per batch
    lens = np.full(len(sub), 64, np.uint32)
    sites = ("nat44_egress", "nat44_ingress", "pipeline_up", "pipeline_tc")

    def frames(flow_set, site):
        return S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), np.uint32(0x08080808), 17,
                              20000 + 100 * flow_set + 10 * site, 53, lens, l4_check=0x1234)

    setup = len(sc.steps)
    seq = 1
    sc.run("nat44_egress", scenarios.fixed(np.concatenate([frames(s, i) for s in (1, 2) for i in range(4)])), np.tile(lens, 8), ns)
    arp = scenarios.fixed(frames(0, 0)[:1])
    arp[12:14] = [0x08, 0x06]

    def replies(res, flow_set):
        out = res[f"s{setup:03d}_frames"].reshape(8, len(sub), 64)[4 * (flow_set - 1) + 1].copy()
        rep = out.copy()
        rep[:, 26:30], rep[:, 30:34] = out[:, 30:34], out[:, 26:30]
        rep[:, 34:36], rep[:, 36:38] = out[:, 36:38], out[:, 34:36]
        return rep

    def touch(flow_set, now):
        nonlocal seq
        for i, prog in enumerate(sites):
            if prog == "nat44_ingress":
                sc.run_from(prog, lambda res, fs=flow_set, t=now + i: {"arena": replies(res, fs).reshape(-1), "lens": lens,
                                                                       "now_ns": t, "stride": 64})
            else:
                sc.run(prog, scenarios.fixed(frames(flow_set, i)), lens, now + i)
        seq += 4

    def filler(count, now):
        nonlocal seq
        sc.repeat("antispoof_ingress", arp, np.full(1, 64, np.uint32), now, count)
        seq += count

    filler(4, 2 * ns)
    first = seq + 1
    touch(1, 3 * ns)
    filler(EPOCH_PERIOD - 5 - seq, 4 * ns)
    touch(2, 5 * ns)
    assert seq + 1 == EPOCH_PERIOD  # the next batch clears the epochs
    touch(2, 6 * ns)
    filler(first + EPOCH_PERIOD - 1 - seq, 7 * ns)
    touch(1, 8 * ns)  # the same epoch values as batches first..first+3
    assert seq == first + EPOCH_PERIOD + 3
    return sc, seq


def test_last_seen_across_the_epoch_wrap(ora_kind):
    """The 16-bit epoch wrap, device-resident as the headline runs, against the oracle: nat_sessions (last_seen
    above all), counters, verdicts and frames."""
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    sc, batches = epoch_wrap_script()
    assert batches > EPOCH_PERIOD
    want = harness.run_script(harness.OracleBackend(ora_kind), sc)
    last_seen = want["tv_nat_sessions"].view(L.nat_session)["last_seen"]
    assert len(last_seen) == 128 and last_seen.min() >= 6 * NS  # every session's last touch is one of the late ones
    gpu = harness.GpuBackend(pinned="device")
    try:
        got = harness.run_script(gpu, sc)
    finally:
        gpu.close()
    harness.compare(want, got, f"epoch wrap: {ora_kind} oracle vs gpu (device-resident)")
