"""Incremental replication (bng_delta_*): a standby context that applies the active context's deltas holds the
active's tables, accounting records and interception targets, and after a failover computes what the active would
have computed."""
import ctypes as C
import errno
import hashlib
import os

import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import Dataplane
from bng_b200 import layouts as L
from bng_b200 import workloads as W
from bng_b200.layouts import as_bytes

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ALL_MAPS = harness.TABLES + harness.STATS_MAPS
UP_PROGS = ("nat44_egress", "qos_ingress_prog", "pipeline_up", "pipeline_tc", "nat44_ingress", "qos_egress_prog")
SMALL = dict(max_subscribers=1 << 14, max_nat_sessions=1 << 16, max_eim_mappings=1 << 16, max_batch=1 << 16,
             event_capacity=1 << 16)


def dumps(dp, maps=ALL_MAPS):
    out = {}
    for m in maps:
        if m in harness.STATS_MAPS:
            out[m] = (np.zeros((1, 4), np.uint8), dp.stats(m).view(np.uint8).reshape(1, -1))
            continue
        k, v = dp.dump(m)
        out[m] = (k, harness.mask_padding(m, v) if len(v) else v)
    return out


def li_targets(dp):
    s = next((s for s in harness.blob_sections(dp.snapshot()) if s.name == "li_targets"), None)
    if s is None:
        return []
    return sorted(zip(s.keys.view("<u4").reshape(-1).tolist(), s.vals.view("<u4").reshape(-1).tolist()))


def acct(dp):
    a, r = dp.acct_dump()
    return a, r.view(np.uint8)


def assert_same(a, b, what, maps=ALL_MAPS):
    da, db = dumps(a, maps), dumps(b, maps)
    for m in maps:
        assert np.array_equal(da[m][0], db[m][0]), f"{what}: {m} keys differ ({len(da[m][0])} vs {len(db[m][0])})"
        assert np.array_equal(da[m][1], db[m][1]), f"{what}: {m} values differ"
    aa, ab = acct(a), acct(b)
    assert np.array_equal(aa[0], ab[0]) and np.array_equal(aa[1], ab[1]), f"{what}: accounting records differ"
    assert li_targets(a) == li_targets(b), f"{what}: interception targets differ"


def ship(a, b, **kw):
    blob = a.delta_export(**kw)
    assert b.delta_apply(blob) == 0
    return blob


class Replicating(harness.GpuBackend):
    """The active context of a script; after every step that changes state its delta (EXACT) goes to the standby
    `peer`, which must then hold the same tables."""

    def __init__(self, peer, pinned, **opts):
        super().__init__(pinned=pinned, **opts)
        self.peer = peer
        self.dp.delta_enable()
        for p in UP_PROGS:
            self.dp.acct_enable(p)
        self.runs = 0

    def _ship(self, what):
        ship(self.dp, self.peer, exact=True)
        assert_same(self.dp, self.peer, what)

    def update(self, m, k, v, flags):
        r = super().update(m, k, v, flags)
        ship(self.dp, self.peer, exact=True)
        return r

    def delete(self, m, k):
        r = super().delete(m, k)
        ship(self.dp, self.peer, exact=True)
        return r

    def run(self, *a, **kw):
        self.runs += 1
        if self.runs == 2:  # targets change between batches
            self.dp.li_target_set(0x6400000A, 7)
            self.dp.li_target_set(0x0300000A, 8)
        if self.runs == 4:
            self.dp.li_target_del(0x6400000A)
        v = super().run(*a, **kw)
        self._ship(f"after run {self.runs}")
        return v

    def run_repeat(self, *a, **kw):
        v = super().run_repeat(*a, **kw)
        self._ship("after a repeated run")
        return v


@pytest.mark.parametrize("feed", [False, "device"], ids=["pageable", "device"])
@pytest.mark.parametrize("script", sorted(scenarios.ALL_SCRIPTS))
def test_exact_replication(script, feed):
    b = Dataplane(**SMALL)
    a = Replicating(b, feed)
    try:
        harness.run_script(a, scenarios.ALL_SCRIPTS[script]())
        assert_same(a.dp, b, f"{script}: end")
        assert b.lru_evictions == 0 and b.delta_info() == a.dp.delta_info()
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("script", ["nat", "pipeline", "qos", "dhcp"])
def test_exact_replication_into_other_capacities(script):
    b = Dataplane(max_subscribers=1 << 12, max_nat_sessions=1 << 13, max_eim_mappings=1 << 13, max_batch=1 << 16)
    a = Replicating(b, False)
    try:
        harness.run_script(a, scenarios.ALL_SCRIPTS[script]())
    finally:
        a.close()
        b.close()


class Failover(harness.GpuBackend):
    """Replicates to the standby until `k` runs have been made; from then on every step runs on both contexts, must give
    the same results on both, and the standby's results are the ones returned (and its tables the ones dumped)."""

    def __init__(self, k, pinned):
        super().__init__(pinned=pinned)
        self.k, self.runs = k, 0
        self.b = harness.GpuBackend(pinned=pinned)
        self.dp.delta_enable()
        self.pending = {m: [] for m in harness.EVENT_MAPS}
        self.live = False

    def close(self):
        super().close()
        self.b.close()

    def _both(self, name, *a):
        if not self.live:
            return getattr(super(), name)(*a)
        ra = getattr(harness.GpuBackend, name)(self, *[x.copy() if isinstance(x, np.ndarray) else x for x in a])
        rb = getattr(self.b, name)(*a)
        assert np.array_equal(np.asarray(ra), np.asarray(rb)), f"{name} after failover: {ra} vs {rb}"
        return rb

    def update(self, *a):
        return self._both("update", *a)

    def delete(self, *a):
        return self._both("delete", *a)

    def lookup(self, m, k):
        if not self.live:
            return super().lookup(m, k)
        va, vb = super().lookup(m, k), self.b.lookup(m, k)
        assert (va is None) == (vb is None) and (va is None or np.array_equal(va, vb))
        return vb

    def _switch(self):
        if self.live or self.runs < self.k:
            return
        ship(self.dp, self.b.dp, exact=True)
        for m in harness.EVENT_MAPS:  # what the active emitted before the failover is drained on the active
            self.pending[m].append(super().drain(m))
        self.live = True

    def run(self, prog, arena, lens, *rest):
        self._switch()
        if not self.live:
            self.runs += 1
            return super().run(prog, arena, lens, *rest)
        a2, l2 = arena.copy(), lens.copy()
        rest2 = [x.copy() if isinstance(x, np.ndarray) else x for x in rest]
        va = harness.GpuBackend.run(self, prog, a2, l2, *rest2)
        vb = self.b.run(prog, arena, lens, *rest)
        assert np.array_equal(va, vb) and np.array_equal(a2, arena) and np.array_equal(l2, lens), "run after failover differs"
        return vb

    def run_repeat(self, prog, arena, lens, now, stride, count):
        self._switch()
        if not self.live:
            self.runs += 1
            return super().run_repeat(prog, arena, lens, now, stride, count)
        a2, l2 = arena.copy(), lens.copy()
        va = harness.GpuBackend.run_repeat(self, prog, a2, l2, now, stride, count)
        vb = self.b.run_repeat(prog, arena, lens, now, stride, count)
        assert np.array_equal(va, vb) and np.array_equal(a2, arena), "repeated run after failover differs"
        return vb

    def drain(self, m):
        if not self.live:
            return super().drain(m)
        ea, eb = super().drain(m), self.b.drain(m)
        assert np.array_equal(harness.mask_padding(m, ea), harness.mask_padding(m, eb)), f"{m} after failover differs"
        out = [e for e in self.pending[m] + [eb] if len(e)]
        self.pending[m] = []
        return np.concatenate(out) if out else eb

    def stats(self, m):
        self._switch()
        return self.b.stats(m) if self.live else super().stats(m)

    def dump(self, m):
        self._switch()
        if not self.live:
            return super().dump(m)
        ka, va = super().dump(m)
        kb, vb = self.b.dump(m)
        assert np.array_equal(ka, kb) and np.array_equal(harness.mask_padding(m, va), harness.mask_padding(m, vb)), m
        return kb, vb

    def health(self):
        return {"lru_overflow": self.b.dp.lru_overflow, "events_lost": self.b.dp.events_lost,
                "standby_lru_evictions": self.b.dp.lru_evictions}


@pytest.mark.parametrize("feed", [False, "device"], ids=["pageable", "device"])
@pytest.mark.parametrize("script", ["nat", "nat_parity", "nat_stale", "nat_exhaust", "pipeline", "pipeline_tc", "qos",
                                    "ticks", "ipopts", "dhcp"])
def test_failover_equivalence(script, feed):
    """After k batches the standby takes over; from then on both contexts give the same verdicts, frames, lengths, event
    records and tables, and the standby's results are the goldens'."""
    gold = harness.load_golden(os.path.join(GOLD, script + ".npz"))
    for k in (1, 3):
        be = Failover(k, feed)
        try:
            res = harness.run_script(be, scenarios.ALL_SCRIPTS[script]())
        finally:
            be.close()
        harness.compare(gold, res, f"{script}: golden vs standby after a failover at run {k}")


VOLATILE = {  # (byte ranges of the ABI value that are counters or stamps, the time field (offset, size))
    "nat_sessions": ([(40, 32)], (24, 8)),
    "eim_table": ([], (16, 8)),
    "qos_ingress": ([(0, 8)], (8, 8)),
    "qos_egress": ([(0, 8)], (8, 8)),
}


def _by_key(keys, vals):
    return {bytes(k): v for k, v in zip(keys, vals)}


def test_thresholded_mode():
    T = 5 * 10**9
    b = Dataplane(**SMALL)
    a = harness.GpuBackend()
    a.dp.delta_enable()

    class Probe(harness.GpuBackend):
        def run(self, *x, **kw):
            v = harness.GpuBackend.run(self, *x, **kw)
            ship(self.dp, b, refresh_ns=T)
            da, db = dumps(self.dp, harness.TABLES), dumps(b, harness.TABLES)
            for m in harness.TABLES:
                assert np.array_equal(da[m][0], db[m][0]), m
                vol, tf = VOLATILE.get(m, ([], None))
                if tf is None:
                    assert np.array_equal(da[m][1], db[m][1]), m
                    continue
                va, vb = da[m][1].copy(), db[m][1].copy()
                ta, tb = (x[:, tf[0]:tf[0] + 8].copy().view("<u8").reshape(-1) for x in (va, vb))
                assert np.all(ta >= tb) and np.all(ta - tb <= T), f"{m}: time fields more than T apart"
                for off, n in vol:
                    ca, cb = (x[:, off:off + n].copy().view("<u8") for x in (va, vb))
                    if m == "nat_sessions":
                        assert np.all(ca >= cb), f"{m}: the standby's counters are ahead"
                for off, n in vol + [tf]:
                    va[:, off:off + n] = 0
                    vb[:, off:off + n] = 0
                assert np.array_equal(va, vb), f"{m}: non-volatile bytes differ"
            return v

    p = Probe(dp=a.dp)
    try:
        harness.run_script(p, scenarios.ALL_SCRIPTS["nat"]())
    finally:
        a.close()
        b.close()


def _load(dp, wl):
    for m, k, v in wl.maps:
        assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
    for prog, h, l in wl.prewarm:
        dp.run(prog, h.reshape(-1).copy(), l.copy(), wl.now0 - 1, stride=64)


def test_thresholded_steady_traffic_sends_no_sessions():
    n = 1 << 16
    wl = W.build("nat_steady_64", n)
    a, b = Dataplane(max_batch=n, **W.sizing(wl)), Dataplane(max_batch=n, **W.sizing(wl))
    try:
        a.delta_enable()
        _load(a, wl)
        a.run(wl.prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0, stride=64)
        ship(a, b, refresh_ns=10**9)
        for i in range(1, 5):
            a.run(wl.prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0 + i * wl.now_step, stride=64)
            blob = ship(a, b, refresh_ns=10**9)
            _, sec = L.parse_delta(blob)
            assert sec["nat_sessions"][2].shape[0] == 0 and sec["nat_sessions"][1].shape[0] == 0, i
        blob = ship(a, b, exact=True)
        assert L.parse_delta(blob)[1]["nat_sessions"][2].shape[0] > 0
        assert_same(a, b, "steady traffic, then an exact delta")
    finally:
        a.close()
        b.close()


def _nat_setup(dp, n_subs=20, pps=64):
    sc = harness.Script("maps")
    scenarios.nat_maps(sc, n_subs, pps, 0x0F)
    for st in sc.steps:
        assert dp.update_batch(st[1], st[2], st[3], st[4]) == 0


def _frames(n_subs, n_flows, base_port):
    from test_gpu_flush import _frames as ff
    sub = np.repeat(np.arange(n_subs), n_flows)
    lens = np.full(len(sub), 64, np.uint32)
    return ff(sub, (base_port + np.tile(np.arange(n_flows), n_subs)).astype(np.uint32), lens), lens


def test_churn():
    NS = 10**9
    opts = dict(max_subscribers=1 << 10, max_nat_sessions=256, max_eim_mappings=256, max_batch=1 << 12)
    a, b = Dataplane(**opts), Dataplane(**opts)
    try:
        a.delta_enable()
        for p in UP_PROGS:
            a.acct_enable(p)
        _nat_setup(a)
        ship(a, b, exact=True)
        assert_same(a, b, "maps")
        # LRU eviction at capacity, and the rebuild once evictions pass a quarter of the slots
        r0, now = a.table_rebuilds, 10 * NS
        for i in range(6):
            h, lens = _frames(20, 16, 2000 + 16 * i)
            a.run("nat44_egress", h.reshape(-1).copy(), lens, now + i * NS, stride=64)
            ship(a, b, exact=True)
            assert_same(a, b, f"eviction round {i}")
        assert a.lru_evictions > 0 and a.table_rebuilds > r0
        assert b.lru_evictions == 0
        # expiry sweep, flush
        a.sweep(now + 400 * NS)
        ship(a, b, exact=True)
        assert_same(a, b, "sweep")
        h, lens = _frames(20, 8, 9000)
        a.run("nat44_egress", h.reshape(-1).copy(), lens, now + 401 * NS, stride=64)
        subs = a.dump("subscriber_nat")[0].copy().view("<u4").reshape(-1)
        a.nat_flush(subs[:5], now + 402 * NS)
        ship(a, b, exact=True)
        assert_same(a, b, "flush")
        # staged upserts, clear, restore
        k, v = a.dump("subscriber_nat")
        v2 = v.copy()
        v2[:, 8] ^= 1
        for i in range(3):
            a.update_staged("subscriber_nat", k[i], v2[i])
        ship(a, b, exact=True)
        assert_same(a, b, "staged upserts")
        snap = a.snapshot()
        assert a.clear("nat_reverse") == 0 and a.clear("subscriber_nat") == 0
        ship(a, b, exact=True)
        assert_same(a, b, "clear")
        a.restore(snap)
        ship(a, b, exact=True)
        assert_same(a, b, "restore")
        assert b.lru_evictions == 0
    finally:
        a.close()
        b.close()


def test_protocol_and_errors():
    from bng_b200.dataplane import load_library
    lib = load_library()
    a, b, c = Dataplane(**SMALL), Dataplane(**SMALL), Dataplane(**SMALL)
    try:
        n = C.c_uint64(0)
        assert lib.bng_delta_export(a.h, 0, 0, None, 0, C.byref(n)) == -errno.EINVAL  # not enabled
        a.delta_enable()
        assert lib.bng_delta_export(a.h, 0, 4, None, 0, C.byref(n)) == -errno.EINVAL  # unknown flag
        assert b.lib.bng_delta_apply(b.h, b"garbage" * 10, 70) == -errno.EINVAL
        be = harness.GpuBackend(dp=a)
        sc = scenarios.ALL_SCRIPTS["nat"]()
        steps = sc.steps
        blobs = []
        for st in steps:  # the first half of the script, one delta after every run
            if st[0] == "update":
                be.update(st[1], st[2], st[3], st[4])
            elif st[0] == "run":
                be.run(st[1], st[2].copy(), st[3].copy(), st[4], st[5], st[6], st[7])
                blobs.append(a.delta_export())
            if len(blobs) == 4:
                break
        h0 = L.parse_delta(blobs[0])[0]
        assert h0["flags"] & 1 and h0["seq_from"] == 0 and h0["seq_to"] == 1  # the first export is FULL
        # a gap: nothing changes
        assert b.delta_apply(blobs[1]) == -errno.ESTALE and b.map_info("nat_sessions")["count"] == 0
        assert b.delta_apply(blobs[0]) == 0
        before = dumps(b)
        assert b.delta_apply(blobs[2]) == -errno.ESTALE
        after = dumps(b)
        assert all(np.array_equal(before[m][1], after[m][1]) for m in before)
        assert b.delta_apply(blobs[1]) == 0 and b.delta_apply(blobs[2]) == 0 and b.delta_info() == (h0["stream_id"], 3)
        # a foreign stream
        c.delta_enable()
        c.delta_export()
        assert b.delta_apply(c.delta_export()) == -errno.ESTALE
        # FULL re-synchronises (after the missed blobs[3])
        assert b.delta_apply(a.delta_export(exact=True)) == -errno.ESTALE
        assert b.delta_apply(a.delta_export(full=True, exact=True)) == 0
        assert_same(a, b, "FULL")
        # a FULL delta into a fresh context is a restore of a snapshot
        d = Dataplane(**SMALL)
        e = Dataplane(**SMALL)
        try:
            full = a.delta_export(full=True, exact=True)
            assert d.delta_apply(full) == 0 and b.delta_apply(full) == 0
            e.restore(a.snapshot())
            assert_same(d, e, "FULL vs restore")
        finally:
            d.close()
            e.close()
        # -ENOSPC sizes the blob and leaves the baseline: the same changes come with the next call
        h, lens = _frames(5, 4, 7000)
        a.run("nat44_egress", h.reshape(-1).copy(), lens, 99 * 10**9, stride=64)
        buf = C.create_string_buffer(64)
        assert lib.bng_delta_export(a.h, 0, 2, buf, 64, C.byref(n)) == -errno.ENOSPC and n.value > 64
        need = n.value
        _, s0 = a.delta_info()
        blob = a.delta_export(exact=True)
        assert len(blob) == need and L.parse_delta(blob)[0]["seq_from"] == s0
        assert b.delta_apply(blob) == 0
        assert_same(a, b, "after -ENOSPC")
        # disabling frees tracking; the export refuses
        a.delta_enable(False)
        assert lib.bng_delta_export(a.h, 0, 0, None, 0, C.byref(n)) == -errno.EINVAL
    finally:
        a.close()
        b.close()
        c.close()


def test_tracking_adds_no_launches_to_batches():
    wl = W.build("pipeline_64", 1 << 14)
    dp = Dataplane(max_batch=1 << 14, **W.sizing(wl))
    try:
        _load(dp, wl)

        def per_run():
            l0 = dp.launch_count
            dp.run(wl.prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0, stride=64)
            return dp.launch_count - l0

        off = per_run()
        dp.delta_enable()
        on = per_run()
        dp.delta_export()
        assert per_run() == on == off
        l0 = dp.launch_count
        dp.delta_export()
        assert dp.launch_count > l0  # the export's own kernels
    finally:
        dp.close()


def test_scale_reference_capacities():
    """2^20 nat_cold frames into tables of the reference's sizes (4 M sessions, 2 M EIM mappings, 1 M subscribers),
    replicated exactly: a FULL delta, then an incremental one after a second batch."""
    n = 1 << 20
    wl = W.build("nat_cold_64", n)
    a, b = Dataplane(max_batch=n), Dataplane(max_batch=n)
    try:
        a.delta_enable()
        _load(a, wl)
        a.run(wl.prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0, stride=64)
        ship(a, b, exact=True)
        assert_same(a, b, "2^20 frames, FULL")
        a.run(wl.prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0 + wl.now_step, stride=64)
        ship(a, b, exact=True)
        assert_same(a, b, "2^20 frames, incremental")
        assert a.map_info("nat_sessions")["count"] > 500_000 and b.lru_evictions == 0
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("world", [2, 8])
def test_sharded_replication(world):
    """Each shard replicates to its own peer; the union of the peers' tables is the union of the actives'."""
    n = 1 << 14
    act, peers = [], []
    try:
        for r in range(world):
            wl = W.build("pipeline_imix", n, r, world)
            a, b = Dataplane(max_batch=n, **W.sizing(wl)), Dataplane(max_batch=n, **W.sizing(wl))
            act.append(a), peers.append(b)
            a.delta_enable()
            _load(a, wl)
            from bng_b200.workloads import slot16
            off16, stride, g = slot16(wl.lens, wl.imix, wl.headers.shape[1])
            arena = np.zeros(g * 16 + 64, np.uint8) if off16 is not None else wl.headers.reshape(-1).copy()
            if off16 is not None:
                for i in range(wl.n):
                    arena[off16[i] * 16:off16[i] * 16 + wl.headers.shape[1]] = wl.headers[i]
            a.run(wl.prog, arena, wl.lens.copy(), wl.now0, off16=off16, stride=stride)
            ship(a, b, exact=True)
            a.run(wl.prog, arena, wl.lens.copy(), wl.now0 + wl.now_step, off16=off16, stride=stride)
            ship(a, b, exact=True)
        for m in ("nat_sessions", "nat_reverse", "eim_table", "subscriber_nat", "qos_ingress"):
            ua = np.concatenate([x.dump(m)[0] for x in act])
            ub = np.concatenate([x.dump(m)[0] for x in peers])
            assert len(ua) > 0 and np.array_equal(np.unique(ua, axis=0), np.unique(ub, axis=0)), m
        for a, b in zip(act, peers):
            assert_same(a, b, f"shard of {world}")
    finally:
        for x in act + peers:
            x.close()


# ---------------------------------------------------------------------------
# the three state blobs of one richly configured context, section by section
# ---------------------------------------------------------------------------
BLOB_SECTIONS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "blob_sections.json")


def _rich():
    """A context with a section of every kind: pipeline_up state, accounting and idle records, interception targets,
    IPv6 prefixes and ND bindings."""
    from bng_b200 import synth as S
    from test_gpu_move import _small
    dp, _, ips = _small(n_subs=40)
    v6 = np.zeros((20, 16), np.uint8)
    v6[:, :4] = [0x20, 0x01, 0x0D, 0xB8]
    v6[:, 5] = np.arange(20)
    assert dp.ipv6_prefixes_set(v6, [56] * 20, ips[:20]) == 0
    nd = np.zeros(20, L.bng_nd_binding)
    nd["prefix"], nd["prefix_len"], nd["pio_flags"] = v6, 64, 0xC0
    nd["valid_lft"], nd["preferred_lft"], nd["expires_s"] = 7200, 3600, 2_000_000
    assert dp.update_batch("nd_bindings", S.sub_mac_key(np.arange(20)), nd) == 0
    return dp, ips, S.sub_mac_key(np.arange(len(ips)))


def _section_list(secs):
    """(name, kind, key_size, value_size, n_del, count, digest of the sorted rows) per section, in blob order."""
    out = []
    for s in secs:
        rows = sorted(bytes(r) for r in np.concatenate([s.keys, harness.mask_padding(s.name, s.vals)], axis=1))
        h = hashlib.sha256(b"".join(sorted(bytes(r) for r in s.dels)) + b"|" + b"".join(rows)).hexdigest()[:16]
        out.append([s.name, s.kind, s.keys.shape[1], s.vals.shape[1], len(s.dels), len(s.keys), h])
    return out


def blob_section_lists():
    """The section lists of a snapshot, a FULL delta and a hand-over export of every other subscriber."""
    dp, ips, macs = _rich()
    try:
        snap = harness.blob_sections(dp.snapshot())
        dp.delta_enable()
        delta = harness.blob_sections(dp.delta_export(full=True), L.delta_header.itemsize, with_del=True)
        move = harness.blob_sections(dp.sub_export(ips[1::2], macs[::2]))
        return {"snapshot": _section_list(snap), "delta": _section_list(delta), "sub_export": _section_list(move)}
    finally:
        dp.close()


def test_blob_sections_are_pinned():
    """Section order, headers and contents of all three blobs, as the library wrote them before their framing was
    shared (tests/golden/blob_sections.json)."""
    import json
    with open(BLOB_SECTIONS) as f:
        want = json.load(f)
    got = blob_section_lists()
    for producer in want:
        assert [s[:6] for s in got[producer]] == [s[:6] for s in want[producer]], producer
        assert got[producer] == want[producer], f"{producer}: rows differ"


def test_restore_refuses_a_wrapping_section_whole():
    """A snapshot whose second section claims 2^61 four-byte keys and values, so that count * (key_size + value_size)
    wraps to 0, is refused before anything changes: not even the valid first section is loaded into its emptied map."""
    dp, ips, _ = _rich()
    try:
        blob = dp.snapshot()
        secs = harness.blob_sections(blob)
        bad_hdr = np.zeros(1, L.delta_section)
        bad_hdr["name"], bad_hdr["kind"], bad_hdr["key_size"], bad_hdr["value_size"] = b"subscriber_idle", 7, 4, 4
        bad_hdr["n_up"] = 1 << 61
        bad = blob[:8] + (2).to_bytes(8, "little") + blob[16:secs[1].start] + bad_hdr.tobytes() + bytes(64)
        assert secs[0].name == "subscriber_bindings" and len(secs[0].keys)
        dp.clear("subscriber_bindings")
        before = dumps(dp), acct(dp), li_targets(dp), dp.idle_read(ips)
        assert dp.lib.bng_restore(dp.h, bad, len(bad)) == -errno.EINVAL
        after = dumps(dp), acct(dp), li_targets(dp), dp.idle_read(ips)
        for m in ALL_MAPS:
            assert np.array_equal(before[0][m][0], after[0][m][0]) and np.array_equal(before[0][m][1], after[0][m][1]), m
        assert all(np.array_equal(x, y) for x, y in zip(before[1] + before[3], after[1] + after[3]))
        assert before[2] == after[2] and len(before[2]) == 2
    finally:
        dp.close()
