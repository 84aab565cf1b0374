"""Lawful intercept (bng_li_*): the GPU's records against the rule of include/bng_b200.h, restated here from the
oracle's inputs and outputs alone, on the pageable, pinned and device feeds.

The rule: upstream programs capture a frame whose IPv4 source, as it entered, is a target (untagged Ethernet II,
ethertype 0x0800, bytes 26-29 present), with the bytes it entered with; downstream programs a frame whose destination,
as it leaves, is a target (bytes 30-33), with the bytes it leaves with.  The verdict is TC_ACT_OK or TC_ACT_SHOT; in
the pipelines a frame antispoof_ingress drops is not captured.  cap_len = min(len, bytes in the frame's storage,
snaplen); records drain ordered by (batch, frame)."""
import errno

import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import dataplane as D
from bng_b200 import layouts as L
from bng_b200 import synth as S
from bng_b200 import workloads as W
from bng_b200.layouts import as_bytes

pytestmark = pytest.mark.gpu

UP = ("nat44_egress", "qos_ingress_prog", "pipeline_up", "pipeline_tc")
DOWN = ("nat44_ingress", "qos_egress_prog")
PIPES = ("pipeline_up", "pipeline_tc")
FEEDS = [False, True, "device"]
FEED_IDS = ["pageable", "pinned", "device"]
SCRIPTS = [s for s in sorted(scenarios.ALL_SCRIPTS) if s not in ("antispoof", "dhcp")]
HDR = [f for f in L.bng_li_record.names if f != "pad"]


# ---------------------------------------------------------------------------
# the rule, restated
# ---------------------------------------------------------------------------
def _layout(arena, lens, off16, stride):
    """(start offsets, bytes present in each frame's storage, arena padded so that reads past the end are zeros)."""
    n = len(lens)
    starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(n, dtype=np.int64) * stride
    have = lens.astype(np.int64) if off16 is not None else np.minimum(lens.astype(np.int64), stride)
    return starts, have, np.concatenate([np.asarray(arena, np.uint8).reshape(-1), np.zeros(64, np.uint8)])


def _u32_at(a, starts, off):
    return np.ascontiguousarray(np.stack([a[starts + off + k] for k in range(4)], axis=1)).view("<u4").reshape(-1)


def spec_records(prog, arena_in, frames_out, lens, off16, stride, verdict, now, now_v, targets, batch, snaplen,
                 spoof_drop=None):
    """The records one run gives: a list of (header dict, bytes), in frame order.  targets: {addr: id};
    spoof_drop: bool[n] of the frames antispoof_ingress drops (pipelines)."""
    if prog not in UP + DOWN or not targets:
        return []
    up = prog in UP
    starts, have, a = _layout(arena_in if up else frames_out, lens, off16, stride)
    et = (a[starts + 12] == 0x08) & (a[starts + 13] == 0x00)
    addr = _u32_at(a, starts, 26 if up else 30)
    ok = (have >= (30 if up else 34)) & et & np.isin(addr, np.array(sorted(targets), "<u4"))
    ok &= (verdict == L.TC_ACT_OK) | (verdict == L.TC_ACT_SHOT)
    if prog in PIPES:
        ok &= ~spoof_drop
    out = []
    for i in np.nonzero(ok)[0]:
        cl = int(min(int(lens[i]), int(have[i]), snaplen))
        h = dict(ts_ns=int(now_v[i]) if now_v is not None else int(now), batch=batch, frame=int(i),
                 target_id=targets[int(addr[i])], addr=int(addr[i]), wire_len=int(lens[i]), cap_len=cl,
                 dir=L.LI_UPLINK if up else L.LI_DOWNLINK, verdict=int(verdict[i]), prog=D.PROGRAMS.index(prog))
        out.append((h, a[starts[i]:starts[i] + cl].copy()))
    return out


def got_records(hdr, data):
    assert (hdr["pad"] == 0).all(), "padding of a record is not zero"
    return [({f: int(h[f]) for f in HDR}, d) for h, d in zip(hdr, data)]


def assert_records_equal(got, want, what):
    assert len(got) == len(want), f"{what}: {len(got)} records, the rule gives {len(want)}"
    for k, ((gh, gd), (wh, wd)) in enumerate(zip(got, want)):
        assert gh == wh, f"{what}: record {k}: {gh} vs {wh}"
        assert np.array_equal(gd, wd), f"{what}: record {k} (frame {wh['frame']}): captured bytes differ"


class LiBackend(harness.GpuBackend):
    """The GPU backend with a schedule of target changes before given runs, draining the records after each run."""

    def __init__(self, schedule, pinned, snaplen=0, capacity=0, **opts):
        super().__init__(pinned=pinned, **opts)
        self.schedule, self.runs, self.records = schedule, 0, []
        self.dp.li_configure(snaplen, capacity)

    def run(self, prog, arena, lens, now, off16, stride, prio, now_v=None):
        for op in self.schedule.get(self.runs, ()):
            if op[0] == "set":
                self.dp.li_target_set(op[1], op[2])
            else:
                assert self.dp.li_target_del(op[1]) == 0
        self.runs += 1
        v = super().run(prog, arena, lens, now, off16, stride, prio, now_v)
        self.records.append(got_records(*self.dp.li_drain()))
        return v


def _run_inputs(st, want):
    if st[0] == "run_from":
        d = st[2](want)
        return (st[1], d["arena"], d["lens"].astype(np.uint32), d.get("off16"), int(d.get("stride", 0)), int(d["now_ns"]),
                d.get("now_v"))
    _, prog, arena, lens, now, off16, stride, _, now_v = st
    return prog, arena, lens, off16, stride, now, now_v


def script_targets(script, want):
    """Every address a run of the script carries where interception looks (upstream sources, downstream
    destinations), and one no frame carries."""
    seen = set()
    for si, st in enumerate(script.steps):
        if st[0] not in ("run", "run_from"):
            continue
        prog, arena, lens, off16, stride, _, _ = _run_inputs(st, want)
        if prog in UP + DOWN:
            starts, _, a = _layout(arena if prog in UP else want[f"s{si:03d}_frames"], lens, off16, stride)
            seen |= set(int(x) for x in _u32_at(a, starts, 26 if prog in UP else 30))
    seen.add(0x0A0B0C0D)
    return sorted(seen)[:3000]


def make_schedule(addrs, n_runs, seed=7):
    """All addresses from the first run; from the middle run on a third of them are gone, and a target id is
    replaced; two runs later they come back with new ids."""
    r = np.random.Generator(np.random.PCG64(seed))
    ids = {a: int(x) for a, x in zip(addrs, r.integers(1, 1 << 32, len(addrs)))}
    sched = {0: [("set", a, ids[a]) for a in addrs]}
    mid = max(1, n_runs // 2)
    gone = addrs[::3]
    sched.setdefault(mid, []).extend([("del", a) for a in gone])
    if len(addrs) > 1:
        sched[mid].append(("set", addrs[1], 0xFEEDF00D))
    sched.setdefault(mid + 2, []).extend([("set", a, ids[a] ^ 0x5A5A5A5A) for a in gone])
    return sched


def expected_script_records(script, want, ora_kind, schedule, snaplen=1518):
    """The records of every run of `script`, given the oracle's results and the target schedule."""
    rep = harness.OracleBackend(ora_kind)  # map commands, and antispoof_ingress over the pipelines' frames
    targets, out, runs = {}, [], 0
    try:
        for si, st in enumerate(script.steps):
            if st[0] == "update":
                rep.update(st[1], st[2], st[3], st[4])
                continue
            if st[0] == "delete":
                rep.delete(st[1], st[2])
                continue
            if st[0] not in ("run", "run_from"):
                continue
            for op in schedule.get(runs, ()):
                if op[0] == "set":
                    targets[op[1]] = op[2]
                else:
                    del targets[op[1]]
            runs += 1
            prog, arena, lens, off16, stride, now, now_v = _run_inputs(st, want)
            tag = f"s{si:03d}"
            drop = None
            if prog in PIPES:
                drop = np.asarray(rep.run("antispoof_ingress", arena.copy(), lens.copy(), now, off16, stride, None)) == L.TC_ACT_SHOT
            out.append(spec_records(prog, arena, want[tag + "_frames"], lens, off16, stride, np.asarray(want[tag + "_verdict"]),
                                    now, now_v, dict(targets), runs, snaplen, drop))
    finally:
        rep.close()
    return out


def run_li(script_fn, pinned, ora_kind, schedule, **opts):
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    want = harness.run_script(harness.OracleBackend(ora_kind), script_fn())
    be = LiBackend(schedule, pinned, **opts)
    try:
        got = harness.run_script(be, script_fn())
        harness.compare(want, got, f"{script_fn().name}: {ora_kind} oracle vs gpu with interception on")
    except BaseException:
        be.close()
        raise
    return be, want


def _n_runs(script):
    return sum(st[0] in ("run", "run_from") for st in script.steps)


# ---------------------------------------------------------------------------
# 1. spec parity: every scenario script, every feed
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("script", SCRIPTS)
def test_scenario_records(script, pinned, ora_kind):
    fn = scenarios.ALL_SCRIPTS[script]
    want = harness.run_script(harness.OracleBackend(ora_kind), fn()) if ora_kind != "none" else None
    if want is None:
        pytest.fail("no oracle library present on this box")
    sched = make_schedule(script_targets(fn(), want), _n_runs(fn()))
    be, want = run_li(fn, pinned, ora_kind, sched)
    try:
        exp = expected_script_records(fn(), want, ora_kind, sched)
        assert len(be.records) == len(exp)
        for k, (g, w) in enumerate(zip(be.records, exp)):
            assert_records_equal(g, w, f"{script} ({FEED_IDS[FEEDS.index(pinned)]}) run {k}")
        assert be.dp.li_lost == 0
        flat = [h for run in exp for h, _ in run]
        assert flat, f"{script}: no frame of a target"
        if script.startswith(("nat_exhaust", "pipeline")):
            assert any(h["verdict"] == L.TC_ACT_SHOT for h in flat), f"{script}: no dropped frame was captured"
    finally:
        be.close()


# ---------------------------------------------------------------------------
# 2. boundaries
# ---------------------------------------------------------------------------
def _frames(n, lens, src, dst, proto=17):
    hdr = S.ipv4_headers(np.full(n, 0x020000000001, np.uint64), np.uint64(scenarios.GW_MAC), src, dst,
                         np.full(n, proto, np.uint32), np.full(n, 4000, np.uint32), np.full(n, 53, np.uint32), lens)
    return hdr


def _arena(hdr, lens, stride=None, seed=1):
    """Frames with random payload past their 64-byte header: in an offset-table arena (stride None) or fixed slots."""
    r = np.random.Generator(np.random.PCG64(seed))
    n = len(lens)
    if stride is None:
        sz = ((lens.astype(np.int64) + 15) // 16) * 16
        off = np.concatenate([[0], np.cumsum(sz)[:-1]])
        a = r.integers(0, 256, int(sz.sum()) + 64, dtype=np.uint8)
        for i in range(n):
            a[off[i]:off[i] + 64] = hdr[i]
        return a, (off // 16).astype(np.uint32), 0
    a = r.integers(0, 256, n * stride, dtype=np.uint8).reshape(n, stride)
    a[:, :min(64, stride)] = hdr[:, :min(64, stride)]
    return a.reshape(-1).copy(), None, stride


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("snaplen", [64, 128, 1518])
@pytest.mark.parametrize("stride", [None, 128], ids=["offsets", "stride128"])
def test_snaplen_and_lengths(snaplen, stride, pinned):
    """Lengths 64 to 9000 upstream (qos_ingress_prog) and downstream (qos_egress_prog, which passes frames of an
    address without a bucket unchanged); fixed 128-byte slots hold less than most frames."""
    n = 200
    lens = np.concatenate([np.arange(64, 64 + 100), np.linspace(200, 9000, n - 100).astype(np.int64)]).astype(np.uint32)
    ips = S.sub_ip(np.arange(n) % 4)
    t = {int(x): 100 + k for k, x in enumerate(S.ip_bytes(S.sub_ip(np.arange(3))).view("<u4").reshape(-1))}
    be = harness.GpuBackend(pinned=pinned, max_batch=1 << 12)
    try:
        be.dp.li_configure(snaplen, 1 << 12)
        for a, i in t.items():
            be.dp.li_target_set(a, i)
        for k, (prog, src, dst) in enumerate((("qos_ingress_prog", ips, np.full(n, 0x08080808, np.uint32)),
                                              ("qos_egress_prog", np.full(n, 0x08080808, np.uint32), ips))):
            arena, off16, st = _arena(_frames(n, lens, src, dst), lens, stride, seed=k)
            a, l = arena.copy(), lens.copy()
            v = np.asarray(be.run(prog, a, l, 10**9 + k, off16, st, None))
            assert (v == L.TC_ACT_OK).all() and np.array_equal(a, arena)
            want = spec_records(prog, arena, a, lens, off16, st, v, 10**9 + k, None, t, k + 1, snaplen)
            assert len(want) == 3 * n // 4
            assert_records_equal(got_records(*be.dp.li_drain()), want, f"{prog} snaplen {snaplen}")
        assert be.dp.li_record_size == 64 + (snaplen + 15) // 16 * 16
    finally:
        be.close()


def test_zero_copy_chunk_edges(monkeypatch):
    """A batch of 3 zero-copy chunks (1024 frames each) with targets on both sides of each chunk edge and payload past
    byte 96, and frames with IPv4 options: the pinned feed's records are byte-identical to the pageable and device
    feeds' and to the rule."""
    monkeypatch.setenv("BNG_ZC_CHUNK_LOG2", "10")  # read at bng_open
    n = 3000
    r = np.random.Generator(np.random.PCG64(4))
    lens = r.integers(60, 1600, n).astype(np.uint32)
    sub = np.arange(n) % 50
    hdr = _frames(n, lens, S.sub_ip(sub), np.full(n, 0x08080808, np.uint32))
    opt = np.arange(n) % 7 == 0  # ihl 6: the gather moves the option tail as well
    hdr[opt] = S.ipv4_headers(np.full(opt.sum(), 0x020000000001, np.uint64), np.uint64(scenarios.GW_MAC), S.sub_ip(sub[opt]),
                              np.full(opt.sum(), 0x08080808, np.uint32), np.full(opt.sum(), 17, np.uint32),
                              np.full(opt.sum(), 4000, np.uint32), np.full(opt.sum(), 53, np.uint32), lens[opt], ihl=6)
    arena, off16, _ = _arena(hdr, lens)
    edge = [1022, 1023, 1024, 1025, 2047, 2048, 2049]
    t = {int(x): 7 + k for k, x in enumerate(set(int(y) for y in S.ip_bytes(S.sub_ip(sub[edge])).view("<u4").reshape(-1)))}
    results = []
    for pinned in FEEDS:
        be = harness.GpuBackend(pinned=pinned, max_batch=1 << 12)
        try:
            be.dp.li_configure(0, 1 << 12)
            for a, i in t.items():
                be.dp.li_target_set(a, i)
            for prog in ("qos_ingress_prog", "qos_egress_prog"):
                a, l = arena.copy(), lens.copy()
                be.run(prog, a, l, 10**9, off16, 0, None)
            results.append(got_records(*be.dp.li_drain()))
        finally:
            be.close()
    want = spec_records("qos_ingress_prog", arena, arena, lens, off16, 0, np.zeros(n, np.uint8), 10**9, None, t, 1, 1518)
    assert set(h["frame"] for h, _ in want) >= set(edge) and max(h["cap_len"] for h, _ in want) > 96
    for got, name in zip(results, FEED_IDS):
        assert_records_equal(got[:len(want)], want, f"uplink, {name}")
        assert_records_equal(got, results[0], f"{name} vs pageable")


# ---------------------------------------------------------------------------
# 3. the ring
# ---------------------------------------------------------------------------
def _qos_batch(n, n_subs=8, seed=2):
    lens = np.full(n, 100, np.uint32) + (np.arange(n) % 5).astype(np.uint32)
    hdr = _frames(n, lens, S.sub_ip(np.arange(n) % n_subs), np.full(n, 0x08080808, np.uint32))
    return _arena(hdr, lens, 128, seed)[0], lens


def _all_targets(dp, n_subs=8):
    t = {int(x): k for k, x in enumerate(S.ip_bytes(S.sub_ip(np.arange(n_subs))).view("<u4").reshape(-1))}
    for a, i in t.items():
        dp.li_target_set(a, i)
    return t


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
def test_ring_overflow_keeps_exact_records(pinned):
    n = 2000
    arena, lens = _qos_batch(n)
    be = harness.GpuBackend(pinned=pinned, max_batch=1 << 12)
    try:
        be.dp.li_configure(256, 300)
        t = _all_targets(be.dp)
        kept, want = [], []
        for k in range(3):
            a, l = arena.copy(), lens.copy()
            v = np.asarray(be.run("qos_ingress_prog", a, l, 10**9 + k, None, 128, None))
            want += spec_records("qos_ingress_prog", arena, a, lens, None, 128, v, 10**9 + k, None, t, k + 1, 256)
            if k != 1:  # the second batch finds the ring full of the first's records
                kept += got_records(*be.dp.li_drain())
        assert len(kept) == 600
        by_key = {(h["batch"], h["frame"]): (h, d) for h, d in want}
        for h, d in kept:
            wh, wd = by_key[(h["batch"], h["frame"])]
            assert h == wh and np.array_equal(d, wd)
        assert [(h["batch"], h["frame"]) for h, _ in kept] == sorted((h["batch"], h["frame"]) for h, _ in kept)
        assert len(kept) + be.dp.li_lost == len(want)
    finally:
        be.close()


def test_drain_in_pieces_and_reconfigure():
    n = 500
    arena, lens = _qos_batch(n)
    from bng_b200 import Dataplane
    with Dataplane(max_batch=1 << 12, max_subscribers=1 << 10) as dp:
        assert dp.li_record_size == 0 and dp.li_lost == 0
        t = _all_targets(dp)
        assert dp.li_record_size == 64 + 1520  # the default ring came with the first target
        v = dp.run("qos_ingress_prog", arena.copy(), lens.copy(), 10**9, stride=128)
        want = spec_records("qos_ingress_prog", arena, arena, lens, None, 128, np.asarray(v), 10**9, None, t, 1, 1518)
        got = []
        for cap in (1, 7, 100, 1000):
            h, d = dp.li_drain(cap)
            assert len(h) == min(cap, n - len(got))
            got += got_records(h, d)
        assert_records_equal(got, want, "drained in pieces")
        assert len(dp.li_drain()[0]) == 0
        dp.run("qos_ingress_prog", arena.copy(), lens.copy(), 2 * 10**9, stride=128)
        assert len(dp.li_drain(10)[0]) == 10  # 10 drained, 490 left behind on the host side of the drain
        dp.run("qos_ingress_prog", arena.copy(), lens.copy(), 3 * 10**9, stride=128)  # and 500 in the ring
        dp.li_configure(64, 1 << 10)
        assert dp.li_lost == 990 and dp.li_record_size == 128
        v = dp.run("qos_ingress_prog", arena.copy(), lens.copy(), 4 * 10**9, stride=128)
        h, d = dp.li_drain()
        assert_records_equal(got_records(h, d), spec_records("qos_ingress_prog", arena, arena, lens, None, 128, np.asarray(v),
                                                             4 * 10**9, None, t, 4, 64), "after reconfiguring")


# ---------------------------------------------------------------------------
# 4. cost rule, errors, snapshot
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
def test_no_target_launches_no_kernel(pinned, ora_kind):
    counts = []
    for mode in ("never", "configured", "emptied"):
        be = harness.GpuBackend(pinned=pinned)
        try:
            if mode != "never":
                be.dp.li_configure()
            if mode == "emptied":
                be.dp.li_target_set(0x0100A8C0, 1)
                assert be.dp.li_target_del(0x0100A8C0) == 0
            for name in ("pipeline", "nat", "qos"):
                harness.run_script(be, scenarios.ALL_SCRIPTS[name]())
            counts.append(be.dp.launch_count)
            assert len(be.dp.li_drain()[0]) == 0
        finally:
            be.close()
    assert counts[0] == counts[1] == counts[2], counts


def test_error_codes():
    from bng_b200 import Dataplane
    lib = D.load_library()
    n = D.C.c_uint64(0)
    assert lib.bng_li_configure(None, 0, 0) == -errno.EINVAL
    assert lib.bng_li_target_set(None, 1, 1) == -errno.EINVAL
    assert lib.bng_li_target_del(None, 1) == -errno.EINVAL
    assert lib.bng_li_drain(None, None, 0, D.C.byref(n)) == -errno.EINVAL
    assert lib.bng_li_record_size(None) == 0 and lib.bng_li_lost(None) == 0
    with Dataplane(max_batch=1 << 10, max_subscribers=1 << 10) as dp:
        assert dp.li_target_del(5) == -errno.ENOENT  # nothing allocated yet
        assert lib.bng_li_drain(dp.h, None, 0, D.C.byref(n)) == 0 and n.value == 0
        assert lib.bng_li_drain(dp.h, None, 0, None) == -errno.EINVAL
        assert lib.bng_li_drain(dp.h, None, 5, D.C.byref(n)) == -errno.EINVAL
        assert lib.bng_li_configure(dp.h, 65536, 0) == -errno.EINVAL
        assert lib.bng_li_configure(dp.h, 0, (1 << 30) + 1) == -errno.EINVAL
        assert dp.li_record_size == 0
        for a in range(4096):
            dp.li_target_set(a, a)
        with pytest.raises(D.BngError) as e:
            dp.li_target_set(4096, 1)
        assert e.value.errno == errno.E2BIG
        dp.li_target_set(17, 99)  # replacing an id needs no room
        assert dp.li_target_del(17) == 0 and dp.li_target_del(17) == -errno.ENOENT
        dp.li_target_set(4096, 1)


def _targets_of(dp, addrs, n=64):
    """{addr: id} of the targets in force, observed: one frame per address through qos_ingress_prog."""
    addrs = np.asarray(addrs, np.uint32)
    lens = np.full(len(addrs), 100, np.uint32)
    ips = np.ascontiguousarray(np.asarray(addrs, "<u4")).view(np.uint8).reshape(-1, 4)
    numeric = (ips[:, 0].astype(np.uint32) << 24) | (ips[:, 1].astype(np.uint32) << 16) | (ips[:, 2].astype(np.uint32) << 8) | ips[:, 3]
    hdr = _frames(len(addrs), lens, numeric, np.full(len(addrs), 0x08080808, np.uint32))
    dp.li_drain()
    dp.run("qos_ingress_prog", hdr.reshape(-1).copy(), lens, 10**9, stride=64)
    h, _ = dp.li_drain()
    return {int(x["addr"]): int(x["target_id"]) for x in h}


def _strip_section(blob, name):
    import struct
    out = bytearray(blob[:16])
    nmaps = struct.unpack_from("<Q", blob, 8)[0]
    p, kept = 16, 0
    for _ in range(nmaps):
        hname, = struct.unpack_from("40s", blob, p)
        _, ks, vs, _, cnt = struct.unpack_from("<IIIIQ", blob, p + 40)
        end = p + 64 + cnt * (ks + vs)
        if hname.rstrip(b"\0") != name:
            out += blob[p:end]
            kept += 1
        p = end
    assert kept == nmaps - 1, f"the snapshot has no {name} section"
    struct.pack_into("<Q", out, 8, kept)
    return bytes(out)


def test_snapshot_carries_targets():
    from bng_b200 import Dataplane
    addrs = S.ip_bytes(S.sub_ip(np.arange(40))).view("<u4").reshape(-1)
    t = {int(a): 1000 + k for k, a in enumerate(addrs[:30])}
    with Dataplane(max_batch=1 << 10, max_subscribers=1 << 10) as dp:
        for a, i in t.items():
            dp.li_target_set(a, i)
        blob = dp.snapshot()
        with Dataplane(max_batch=1 << 10, max_subscribers=1 << 11) as other:
            assert other.li_record_size == 0
            other.restore(blob)
            assert _targets_of(other, addrs) == t
        stripped = _strip_section(blob, b"li_targets")
        with Dataplane(max_batch=1 << 10, max_subscribers=1 << 11) as other:
            other.li_target_set(int(addrs[35]), 5)
            other.restore(stripped)  # restoring over live targets: the blob's (none) replace them
            assert _targets_of(other, addrs) == {}
        dp.restore(stripped)
        assert _targets_of(dp, addrs) == {}


# ---------------------------------------------------------------------------
# 5. scale: 2^20 frames of pipeline_imix, about 1 % of the subscribers targeted
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
def test_pipeline_imix_at_scale(pinned):
    import torch
    from bng_b200 import MEM_DEVICE, Dataplane
    n = 1 << 20
    wl = W.pipeline(n)
    spoof = (S.splitmix64_array(0xB2000004 + 37, n) % np.uint64(100)) == 0  # workloads.pipeline's forged sources
    dp = Dataplane(max_batch=n, **W.sizing(wl))
    be = harness.GpuBackend(dp, pinned=pinned)
    try:
        for m, k, v in wl.maps:
            assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
        for prog, h, l in wl.prewarm:
            dp.run(prog, h.reshape(-1).copy(), l.copy(), wl.now0 - 1, stride=64)
        off16, stride, total16 = W.slot16(wl.lens, wl.imix, wl.headers.shape[1], 64)
        arena = np.random.Generator(np.random.PCG64(3)).integers(0, 256, total16 * 16 + 64, dtype=np.uint8)
        hw = wl.headers.shape[1]
        if off16 is None:
            arena[: n * stride].reshape(n, stride)[:, :hw] = wl.headers
        else:
            idx = off16.astype(np.int64)[:, None] * 16 + np.arange(hw)[None, :]
            arena[idx.reshape(-1)] = wl.headers.reshape(-1)
        src = wl.headers[:, 26:30].copy().view("<u4").reshape(-1)
        subs = S.ip_bytes(S.sub_ip(np.arange(0, 10_000, 100))).view("<u4").reshape(-1)  # 100 of the 10 k subscribers
        forged = src[spoof][:20]  # forged sources: addresses of other subscribers, from the wrong MAC
        t = {int(a): k for k, a in enumerate(np.unique(np.concatenate([subs, forged])))}
        dp.li_configure(0, 1 << 17)
        for a, i in t.items():
            dp.li_target_set(a, i)
        a, l = arena[: total16 * 16].copy(), wl.lens.copy()
        v = np.asarray(be.run(wl.prog, a, l, wl.now0, off16, stride, None))
        want = spec_records(wl.prog, arena, a, wl.lens, off16, stride, v, wl.now0, None, t, 2, 1518, spoof_drop=spoof)
        assert 5_000 < len(want) < 1 << 17
        assert np.isin(src[spoof], list(t)).any(), "no forged frame carries a target's source"
        assert_records_equal(got_records(*dp.li_drain()), want, f"pipeline_imix 2^20 ({pinned})")
        assert dp.li_lost == 0
    finally:
        dp.close()
        torch.cuda.synchronize()
