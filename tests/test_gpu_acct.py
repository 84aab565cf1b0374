"""Per-subscriber traffic accounting (bng_acct_*): the GPU's records against the rule of include/bng_b200.h,
restated here from the oracle's inputs and outputs alone, on the pageable, pinned and device feeds.

The rule: a record per address that keys subscriber_nat or qos_ingress when the batch runs.  Upstream programs
charge a frame to the IPv4 source it entered with (untagged Ethernet II, ethertype 0x0800, bytes 26-29 present),
downstream programs to the IPv4 destination it leaves with (bytes 30-33).  TC_ACT_OK counts in the pass pair,
TC_ACT_SHOT in the drop pair; in the pipelines a frame antispoof_ingress drops is not counted.  Bytes are the
frame's len as passed in."""
import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import layouts as L
from bng_b200 import synth as S
from bng_b200 import workloads as W
from bng_b200.layouts import as_bytes
from test_oracle_fuzz import base_maps_and_frames, fuzz_script

pytestmark = pytest.mark.gpu

UP = ("nat44_egress", "qos_ingress_prog", "pipeline_up", "pipeline_tc")
DOWN = ("nat44_ingress", "qos_egress_prog")
PIPES = ("pipeline_up", "pipeline_tc")
ACCOUNTED = UP + DOWN
FEEDS = [False, True, "device"]
FEED_IDS = ["pageable", "pinned", "device"]
SCRIPTS = [s for s in sorted(scenarios.ALL_SCRIPTS) if s not in ("antispoof", "dhcp")]
FIELDS = L.bng_acct.names


# ---------------------------------------------------------------------------
# the rule, restated
# ---------------------------------------------------------------------------
def _addr_keys(keys):
    return set(int(x) for x in np.ascontiguousarray(keys).view("<u4").reshape(-1)) if len(keys) else set()


def _frame_fields(arena, lens, off16, stride, off):
    """(dlen, ethertype bytes ok, the u32 at `off`) of every frame; dlen is what the slot holds of the frame."""
    n = len(lens)
    starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(n, dtype=np.int64) * stride
    dlen = lens.astype(np.int64) if off16 is not None else np.minimum(lens.astype(np.int64), stride)
    a = np.concatenate([np.asarray(arena, np.uint8).reshape(-1), np.zeros(64, np.uint8)])
    et = (a[starts + 12] == 0x08) & (a[starts + 13] == 0x00)
    b = np.stack([a[starts + off + k] for k in range(4)], axis=1)
    return dlen, et, np.ascontiguousarray(b).view("<u4").reshape(-1)


def expected_records(script, want, ora_kind):
    """{address: [8 ints]} for the addresses with a directory entry at the end of `script`, from the oracle's results
    `want` (harness.run_script), its inputs, and a replay of its map commands for the directory at each batch."""
    rep = harness.OracleBackend(ora_kind)  # map commands only (and antispoof_ingress over the pipelines' frames)
    recs = {}
    try:
        for si, st in enumerate(script.steps):
            tag = f"s{si:03d}"
            if st[0] == "update":
                rep.update(st[1], st[2], st[3], st[4])
                continue
            if st[0] == "delete":
                rep.delete(st[1], st[2])
                continue
            assert st[0] in ("run", "run_from", "lookup", "drain"), st[0]
            if st[0] not in ("run", "run_from"):
                continue
            if st[0] == "run_from":
                d = st[2](want)
                prog, arena, lens = st[1], d["arena"], d["lens"].astype(np.uint32)
                off16, stride, now = d.get("off16"), int(d.get("stride", 0)), int(d["now_ns"])
            else:
                _, prog, arena, lens, now, off16, stride, _, _ = st
            dirset = _addr_keys(rep.dump("subscriber_nat")[0]) | _addr_keys(rep.dump("qos_ingress")[0])
            for a in [a for a in recs if a not in dirset]:
                del recs[a]  # the address lost both entries: its record ended
            if prog not in ACCOUNTED:
                continue
            verdict = np.asarray(want[tag + "_verdict"])
            if prog in UP:
                dlen, et, addr = _frame_fields(arena, lens, off16, stride, 26)
                ok = (dlen >= 30) & et
            else:
                dlen, et, addr = _frame_fields(want[tag + "_frames"], lens, off16, stride, 30)
                ok = (dlen >= 34) & et
            if prog in PIPES:
                a2, l2 = arena.copy(), lens.copy()
                av = np.asarray(rep.run("antispoof_ingress", a2, l2, now, off16, stride, None))
                ok &= av != L.TC_ACT_SHOT
            base = 0 if prog in UP else 4
            for i in np.nonzero(ok & ((verdict == L.TC_ACT_OK) | (verdict == L.TC_ACT_SHOT)))[0]:
                a = int(addr[i])
                if a not in dirset:
                    continue
                r = recs.setdefault(a, [0] * 8)
                j = base + (2 if verdict[i] == L.TC_ACT_SHOT else 0)
                r[j] += 1
                r[j + 1] += int(lens[i])
        final = _addr_keys(rep.dump("subscriber_nat")[0]) | _addr_keys(rep.dump("qos_ingress")[0])
    finally:
        rep.close()
    return {a: recs.get(a, [0] * 8) for a in final}


def _as_dict(addrs, recs):
    return {int(a): [int(r[f]) for f in FIELDS] for a, r in zip(addrs, recs)}


def check_records(dp, expected, what):
    got = _as_dict(*dp.acct_dump())
    assert set(got) == set(expected), f"{what}: {len(set(got) ^ set(expected))} addresses differ between the dump and the directory"
    bad = [a for a in expected if got[a] != expected[a]]
    assert not bad, f"{what}: {len(bad)} records differ, e.g. {bad[0]:#010x}: {got[bad[0]]} vs {expected[bad[0]]}"
    addrs = np.array(sorted(expected), dtype="<u4")
    recs, found = dp.acct_read(addrs)
    assert found.all() and _as_dict(addrs, recs) == {a: expected[a] for a in addrs.tolist()}, f"{what}: acct_read differs"


def run_accounted(script_fn, pinned, ora_kind, enable=ACCOUNTED, **opts):
    """Runs the script on the oracle and on the GPU with accounting enabled for `enable`; every ordinary output must
    still match.  Returns (gpu backend, oracle results); the caller closes the backend."""
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    want = harness.run_script(harness.OracleBackend(ora_kind), script_fn())
    be = harness.GpuBackend(pinned=pinned, **opts)
    try:
        for p in enable:
            be.dp.acct_enable(p)
        got = harness.run_script(be, script_fn())
        harness.compare(want, got, f"{script_fn().name}: {ora_kind} oracle vs gpu with accounting on")
    except BaseException:
        be.close()
        raise
    return be, want


# ---------------------------------------------------------------------------
# 1. every supported program, enabled
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("script", SCRIPTS)
def test_golden_scripts_records(script, pinned, ora_kind):
    fn = scenarios.ALL_SCRIPTS[script]
    be, want = run_accounted(fn, pinned, ora_kind)
    try:
        check_records(be.dp, expected_records(fn(), want, ora_kind), f"{script} ({FEED_IDS[FEEDS.index(pinned)]})")
    finally:
        be.close()


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("seed", [11, 13])
@pytest.mark.parametrize("prog", ACCOUNTED)
def test_fuzz_corpora_records(prog, seed, pinned, ora_kind):
    fn = lambda: fuzz_script(prog, seed)  # noqa: E731
    be, want = run_accounted(fn, pinned, ora_kind)
    try:
        check_records(be.dp, expected_records(fn(), want, ora_kind), f"fuzz {prog} {seed} ({FEED_IDS[FEEDS.index(pinned)]})")
    finally:
        be.close()


# ---------------------------------------------------------------------------
# 2. disabled
# ---------------------------------------------------------------------------
def _all_zero(dp):
    addrs, recs = dp.acct_dump()
    assert len(addrs) > 0
    return all(int(recs[f].sum()) == 0 for f in FIELDS)


@pytest.mark.parametrize("enable", [(), ("nat44_ingress", "qos_egress_prog")], ids=["default", "other-programs"])
def test_disabled_programs_count_nothing(enable, ora_kind):
    be, _ = run_accounted(scenarios.ALL_SCRIPTS["pipeline"], False, ora_kind, enable=enable)
    try:
        assert _all_zero(be.dp)
    finally:
        be.close()


def test_enable_error_codes():
    import errno
    from bng_b200 import Dataplane, BngError
    with Dataplane(max_subscribers=1 << 10, max_batch=1 << 10) as dp:
        for p in ("antispoof_ingress", "nat44_hairpin_xdp", "dhcp_fastpath_prog"):
            with pytest.raises(BngError) as e:
                dp.acct_enable(p)
            assert e.value.errno == errno.EOPNOTSUPP
        for p in (-1, 9, 1 << 20):
            with pytest.raises(BngError) as e:
                dp.acct_enable(p)
            assert e.value.errno == errno.EINVAL
        dp.acct_enable("pipeline_up", False)  # disabling what was never enabled


# ---------------------------------------------------------------------------
# 3. lifecycle
# ---------------------------------------------------------------------------
def _qos_frames(ips, n_each, length=100):
    ips = np.repeat(np.asarray(ips, np.uint32), n_each)
    n = len(ips)
    lens = np.full(n, length, np.uint32)
    hdr = S.ipv4_headers(np.full(n, 0x020000000001, np.uint64), np.uint64(scenarios.GW_MAC), ips,
                         np.full(n, 0x08080808, np.uint32), np.full(n, 17, np.uint32), np.full(n, 4000, np.uint32),
                         np.full(n, 53, np.uint32), lens)
    return hdr.reshape(-1).copy(), lens


def _unlimited(n):
    return np.zeros(n, L.token_bucket)


def _rec(dp, ip):
    r, found = dp.acct_read(np.array([ip], "<u4").view(np.uint8).reshape(1, 4))
    return (int(r[0]["up_packets"]), int(r[0]["up_bytes"])) if found[0] else None


def test_lifecycle_of_a_record():
    from bng_b200 import Dataplane
    ips = S.sub_ip(np.arange(32))
    keys = S.ip_bytes(ips)
    with Dataplane(max_subscribers=32, max_batch=1 << 12) as dp:  # a 64-slot directory: slots are reused
        dp.acct_enable("qos_ingress_prog")
        _, nat_v, _ = S.nat_blocks(32, ports_per_sub=8, port_lo=1024, port_hi=1024 + 8 * 8 - 1)
        assert dp.update_batch("qos_ingress", keys, _unlimited(32)) == 0
        assert dp.update_batch("subscriber_nat", keys[:16], nat_v[:16]) == 0
        a, l = _qos_frames(ips, 3)
        dp.run("qos_ingress_prog", a, l, 10**9, stride=64)
        k0 = int(np.ascontiguousarray(keys[0]).view("<u4")[0])
        k20 = int(np.ascontiguousarray(keys[20]).view("<u4")[0])
        assert _rec(dp, k0) == (3, 300) and _rec(dp, k20) == (3, 300)
        # one of the two entries goes: the record stays
        assert dp.delete("qos_ingress", keys[0]) == 0
        assert _rec(dp, k0) == (3, 300)
        assert dp.update("qos_ingress", keys[0], _unlimited(1)) == 0  # and comes back: still the same record
        assert _rec(dp, k0) == (3, 300)
        # both go, then the address comes back: zero
        assert dp.delete("qos_ingress", keys[20]) == 0
        assert _rec(dp, k20) is None
        assert dp.update("qos_ingress", keys[20], _unlimited(1)) == 0
        assert _rec(dp, k20) == (0, 0)
        # bng_map_clear: addresses with a subscriber_nat entry keep their records, the others end
        assert dp.clear("qos_ingress") == 0
        assert _rec(dp, k0) == (3, 300) and _rec(dp, k20) is None
        assert dp.clear("subscriber_nat") == 0
        assert _rec(dp, k0) is None
        assert dp.update_batch("qos_ingress", keys, _unlimited(32)) == 0
        recs, found = dp.acct_read(keys)
        assert found.all() and all(int(recs[f].sum()) == 0 for f in FIELDS)
        # tombstoned slots claimed by other addresses start at zero
        dp.run("qos_ingress_prog", a, l, 2 * 10**9, stride=64)
        for k in keys:
            assert dp.delete("qos_ingress", k) == 0
        others = S.ip_bytes(S.sub_ip(np.arange(100, 132)))
        assert dp.update_batch("qos_ingress", others, _unlimited(32)) == 0
        recs, found = dp.acct_read(others)
        assert found.all() and all(int(recs[f].sum()) == 0 for f in FIELDS)
        # staged upserts are applied before a read (qos_ingress holds 32 entries: one makes room)
        assert dp.delete("qos_ingress", others[0]) == 0
        staged = S.ip_bytes(S.sub_ip(np.array([200])))
        assert dp.update_staged("qos_ingress", staged[0], _unlimited(1)) == 0
        assert dp.acct_read(staged)[1].all()


def test_sweep_eviction_and_rebuild_keep_records():
    """nat44_egress with a small flow table: sessions expire (sweep), are evicted (LRU) and the flow tables are rebuilt;
    the subscriber's record keeps counting through all of it."""
    from bng_b200 import Dataplane
    n_subs = 4
    with Dataplane(max_subscribers=64, max_nat_sessions=64, max_eim_mappings=64, max_batch=1 << 12) as dp:
        sc = harness.Script("setup")
        scenarios.nat_maps(sc, n_subs, 64, 0x0E)
        for st in sc.steps:
            assert dp.update_batch(st[1], st[2], st[3]) == 0
        dp.acct_enable("nat44_egress")
        total = np.zeros((n_subs, 4), np.int64)  # pass packets, pass bytes, drop packets, drop bytes
        r = np.random.Generator(np.random.PCG64(5))
        for step in range(12):
            n = 600
            sub = r.integers(0, n_subs, n)
            sport = (10000 + step * 1000 + r.integers(0, 900, n)).astype(np.uint32)
            lens = np.full(n, 64 + step, np.uint32)
            hdr = S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), np.full(n, 0x08080808, np.uint32),
                                 np.full(n, 17, np.uint32), sport, np.full(n, 53, np.uint32), lens)
            v = dp.run("nat44_egress", hdr.reshape(-1).copy(), lens, (step + 1) * 10**9, stride=64)
            for s in range(n_subs):
                m = sub == s
                total[s] += [int((m & (v == 0)).sum()), int(lens[m & (v == 0)].sum()), int((m & (v == 2)).sum()),
                             int(lens[m & (v == 2)].sum())]
            if step == 5:
                dp.sweep(10**13)  # everything idle for hours: expired
        assert dp.lru_evictions > 0 and dp.table_rebuilds > 0
        recs, found = dp.acct_read(S.ip_bytes(S.sub_ip(np.arange(n_subs))))
        assert found.all()
        got = np.stack([recs["up_packets"], recs["up_bytes"], recs["up_drop_packets"], recs["up_drop_bytes"]], axis=1).astype(np.int64)
        assert np.array_equal(got, total)


# ---------------------------------------------------------------------------
# 4. edges
# ---------------------------------------------------------------------------
def _pipeline_corpus(width=128):
    """The pipeline scenario's map updates and its first batch's frames in fixed `width`-byte slots."""
    updates, frames, lens, now, w = base_maps_and_frames("pipeline")
    frames = np.pad(frames, ((0, 0), (0, max(0, width - w))))[:, :width]
    return updates, frames, np.minimum(lens, width).astype(np.uint32), now, width


def _pipeline_batch(n, seed=3):
    """A pipeline_up script: the pipeline scenario's maps, then one batch of n of its frames."""
    updates, frames, lens, now, stride = _pipeline_corpus()
    idx = np.random.Generator(np.random.PCG64(seed)).integers(0, len(lens), n)

    def fn():
        sc = harness.Script(f"pipeline_{n}")
        sc.steps = list(updates)
        sc.run("pipeline_up", frames[idx].reshape(-1).copy(), lens[idx].copy(), now, stride=stride)
        return sc
    return fn


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("n", [31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 1023, 1024, 1025])
def test_batch_sizes_at_tile_and_chunk_edges(n, pinned, ora_kind, monkeypatch):
    monkeypatch.setenv("BNG_ZC_CHUNK_LOG2", "10")  # zero-copy chunks of 1024 frames (read at bng_open)
    fn = _pipeline_batch(n)
    be, want = run_accounted(fn, pinned, ora_kind)
    try:
        check_records(be.dp, expected_records(fn(), want, ora_kind), f"pipeline_up n={n}")
    finally:
        be.close()


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("prog", ["qos_ingress_prog", "pipeline_up"])
def test_one_subscriber_owns_the_batch(prog, pinned, ora_kind):
    """2^16 frames of one subscriber in one batch (other subscribers' frames around it for the pipeline)."""
    updates, frames, lens, now, stride = _pipeline_corpus()
    n = 1 << 16
    one = frames[np.nonzero(frames[:, 26:30].view("<u4").reshape(-1) == frames[0, 26:30].view("<u4")[0])[0][0]]
    pick = np.zeros(n, np.int64)
    big = np.tile(one, (n, 1))
    ln = np.full(n, 64, np.uint32) + (np.arange(n) % 7).astype(np.uint32)
    if prog == "pipeline_up":
        pick = np.random.Generator(np.random.PCG64(9)).integers(0, len(lens), n)
        mix = np.arange(n) % 5 == 0
        big[mix] = frames[pick[mix]]

    def fn():
        sc = harness.Script(f"one_sub_{prog}")
        sc.steps = list(updates)
        if prog == "qos_ingress_prog":
            sc.update("qos_ingress", one[26:30].reshape(1, 4), _unlimited(1))
        sc.run(prog, big.reshape(-1).copy(), ln.copy(), now, stride=stride)
        return sc
    be, want = run_accounted(fn, pinned, ora_kind, max_batch=n)
    try:
        check_records(be.dp, expected_records(fn(), want, ora_kind), f"{prog}: one subscriber")
    finally:
        be.close()


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
def test_header_split_ring_past_2_pow_32_bytes(pinned):
    """64-byte slots of a header-split ring, len 9000: one subscriber's bytes in one batch exceed 2^32."""
    n = 1 << 19
    ip = S.sub_ip(np.array([7]))
    a, _ = _qos_frames(ip, n)
    lens = np.full(n, 9000, np.uint32)
    be = harness.GpuBackend(pinned=pinned, max_batch=n)
    try:
        assert be.dp.update_batch("qos_ingress", S.ip_bytes(ip), _unlimited(1)) == 0
        be.dp.acct_enable("qos_ingress_prog")
        v = be.run("qos_ingress_prog", a, lens, 10**9, None, 64, None)
        assert (np.asarray(v) == 0).all()
        recs, found = be.dp.acct_read(S.ip_bytes(ip))
        assert found[0] and int(recs[0]["up_packets"]) == n and int(recs[0]["up_bytes"]) == 9000 * n > 1 << 32
    finally:
        be.close()


# ---------------------------------------------------------------------------
# 5. snapshot / restore
# ---------------------------------------------------------------------------
def test_snapshot_carries_records(ora_kind):
    from bng_b200 import Dataplane
    be, _ = run_accounted(scenarios.ALL_SCRIPTS["pipeline"], False, ora_kind)
    try:
        want = _as_dict(*be.dp.acct_dump())
        assert any(sum(r) for r in want.values())
        blob = be.dp.snapshot()
        with Dataplane(max_subscribers=1 << 11, max_nat_sessions=1 << 15, max_eim_mappings=1 << 15, max_batch=1 << 12) as other:
            other.restore(blob)  # another size; accounting never enabled there
            assert _as_dict(*other.acct_dump()) == want
        stripped = harness.strip_section(blob, "subscriber_acct")
        with Dataplane(max_subscribers=1 << 12, max_batch=1 << 12) as other:
            other.acct_enable("pipeline_up")
            other.restore(stripped)
            assert set(_as_dict(*other.acct_dump())) == set(want) and _all_zero(other)
        be.dp.restore(stripped)  # restoring over live records: the blob's (none) replace them
        assert _all_zero(be.dp)
    finally:
        be.close()


# ---------------------------------------------------------------------------
# 6. sharding
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 8])
def test_sharded_records_live_on_the_owner(world):
    from bng_b200 import Dataplane
    n, n_subs, steps = 1 << 16, 1_000, 2
    wl = W.pipeline(n, 0, 1, n_subs=n_subs, flows_per_sub=16, imix=True)
    sub = np.arange(n_subs, dtype=np.uint32)
    ip_shard = {bytes(k): int(s) for k, s in zip(S.ip_bytes(S.sub_ip(sub)), S.shard_of_mac(S.sub_mac_key(sub), world))}
    mac = np.zeros(n, np.uint64)
    for i in range(6):
        mac = (mac << np.uint64(8)) | wl.headers[:, 6 + i].astype(np.uint64)
    frame_shard = S.shard_of_mac(mac, world)
    warm_h, warm_l = wl.prewarm[0][1], wl.prewarm[0][2]
    wmac = np.zeros(len(warm_h), np.uint64)
    for i in range(6):
        wmac = (wmac << np.uint64(8)) | warm_h[:, 6 + i].astype(np.uint64)
    warm_shard = S.shard_of_mac(wmac, world)

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
            dp.acct_enable("pipeline_up")
            mw = (warm_shard == rank) if world_ > 1 else np.ones(len(warm_h), bool)
            dp.run("nat44_egress", warm_h[mw].reshape(-1).copy(), warm_l[mw].copy(), wl.now0 - 1, stride=64)
            mine = np.nonzero(frame_shard == rank)[0] if world_ > 1 else np.arange(n)
            for s in range(steps):
                dp.run(wl.prog, wl.headers[mine].reshape(-1).copy(), wl.lens[mine].copy(), wl.now0 + s * wl.now_step, stride=64)
            return _as_dict(*dp.acct_dump())
        finally:
            dp.close()

    whole = run(0, 1)
    assert sum(sum(r) for r in whole.values()) > 0
    seen = set()
    for rank in range(world):
        part = run(rank, world)
        for a, rec in part.items():
            assert ip_shard[np.array([a], "<u4").tobytes()] == rank, f"{a:#010x} has a record on shard {rank}"
            assert rec == whole[a], f"{a:#010x}: shard {rank} {rec} vs unsharded {whole[a]}"
        seen |= set(part)
    assert seen == set(whole)
