"""Parity at benchmark scale.

* 2^20-frame batches of the BASELINE.json workloads (10 k subscribers, 640 k
  flows, IMIX) against the reference oracle, bit for bit — the oracle finishes
  a million frames in about a second.
* 2^22-frame batches through size-independent properties: the three ways of
  feeding a batch (device-resident, pageable host staging, pinned zero-copy
  pipeline in 2^18-frame chunks) must produce identical bytes, verdicts and
  counters; conservation laws tie the counters to the verdicts.
"""
import numpy as np
import pytest

from bng_b200 import layouts as L
from bng_b200 import synth as S
from bng_b200 import workloads as W
from bng_b200.layouts import as_bytes

pytestmark = pytest.mark.gpu
TABLES = ("nat_sessions", "qos_ingress", "qos_egress", "subscriber_nat", "eim_table", "nat_reverse")


def _load(dp, wl):
    for m, k, v in wl.maps:
        assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m


def _arena(wl, align=64):
    off16, stride, total16 = W.slot16(wl.lens, wl.imix, wl.headers.shape[1], align)
    arena = np.zeros(total16 * 16 + 64, np.uint8)
    hw = wl.headers.shape[1]
    if off16 is None:
        arena[: wl.n * stride].reshape(wl.n, stride)[:, :hw] = wl.headers
    else:
        a16 = arena[: total16 * 16].reshape(total16, 16)
        for g in range(hw // 16):
            a16[off16.astype(np.int64) + g] = wl.headers[:, 16 * g: 16 * g + 16]
    return arena, off16, stride


def _oracle_run(wl, arena, off16, stride, steps):
    from oracle.pyoracle import Oracle, available
    o = Oracle("reference" if available("reference") else "port")
    for m, k, v in wl.maps:
        assert o.update_batch(m, as_bytes(k), as_bytes(v)) == 0
    for prog, h, l in wl.prewarm:
        pa = o.arena(h.shape[0] * 64 + 64)
        pa[: h.shape[0] * 64] = h.reshape(-1)
        o.run(prog, pa, l.copy(), wl.now0 - 1, stride=64)
    outs = []
    for s in range(steps):
        oa = o.arena(len(arena))
        oa[:] = arena
        ol = wl.lens.copy()
        v = o.run(wl.prog, oa, ol, wl.now0 + s * wl.now_step, off16=off16, stride=stride)
        outs.append((v, np.array(oa), ol))
        o.free_arenas()
    stats = {m: o.lookup(m, np.zeros(4, np.uint8)).view("<u8").copy()
             for m in ("antispoof_stats", "qos_stats_map", "nat_stats_map", "stats_map")}
    events = {m: o.drain(m) for m in ("spoof_events", "nat_log_rb")}
    tables = {m: o.dump(m) for m in TABLES}
    return outs, stats, events, tables


def _gpu_run(wl, arena, off16, stride, steps, mode, sizing=None):
    import torch
    from bng_b200 import MEM_DEVICE, MEM_HOST, Dataplane
    dp = Dataplane(max_batch=wl.n, **(sizing or W.sizing(wl)))
    try:
        _load(dp, wl)
        for prog, h, l in wl.prewarm:
            dp.run(prog, h.reshape(-1).copy(), l.copy(), wl.now0 - 1, stride=64)
        outs = []
        for s in range(steps):
            now = wl.now0 + s * wl.now_step
            if mode == "pageable":
                a, l = arena.copy(), wl.lens.copy()
                v = dp.run(wl.prog, a, l, now, off16=off16, stride=stride)
            elif mode == "pinned":
                ta = torch.from_numpy(arena.copy()).pin_memory()
                tl = torch.from_numpy(wl.lens.view(np.int32).copy()).pin_memory()
                to = None if off16 is None else torch.from_numpy(off16.view(np.int32).copy()).pin_memory()
                tv = torch.zeros(wl.n, dtype=torch.uint8).pin_memory()
                dp.run(wl.prog, ta, tl, now, off16=to, stride=stride, verdict=tv, mem=MEM_HOST, arena_bytes=arena.nbytes)
                a, l, v = ta.numpy().copy(), tl.numpy().view(np.uint32).copy(), tv.numpy().copy()
            else:
                ta = torch.from_numpy(arena).cuda()
                tl = torch.from_numpy(wl.lens.view(np.int32)).cuda()
                to = None if off16 is None else torch.from_numpy(off16.view(np.int32)).cuda()
                tv = torch.zeros(wl.n, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()
                dp.run(wl.prog, ta, tl, now, off16=to, stride=stride, verdict=tv, mem=MEM_DEVICE)
                torch.cuda.synchronize()  # not dp.sync(): that runs host-side work a device-path caller never gets
                a, l, v = ta.cpu().numpy(), tl.cpu().numpy().view(np.uint32), tv.cpu().numpy()
            outs.append((np.asarray(v), a, l))
        stats = {m: dp.stats(m) for m in ("antispoof_stats", "qos_stats_map", "nat_stats_map", "stats_map")}
        events = {m: dp.drain(m) for m in ("spoof_events", "nat_log_rb")}
        tables = {m: dp.dump(m) for m in TABLES}
        assert dp.lru_overflow == 0 and dp.events_lost == 0
        return outs, stats, events, tables
    finally:
        dp.close()


def _same(a, b, what):
    (oa, sa, ea, ta), (ob, sb, eb, tb) = a, b
    for s, ((va, aa, la), (vb, ab, lb)) in enumerate(zip(oa, ob)):
        bad = np.nonzero(va != vb)[0]
        assert bad.size == 0, f"{what}: step {s}: {bad.size} verdicts differ, first {bad[:5]}"
        assert np.array_equal(la, lb), f"{what}: step {s}: lengths differ"
        n = min(len(aa), len(ab))
        assert np.array_equal(aa[:n], ab[:n]), f"{what}: step {s}: frame bytes differ at {np.nonzero(aa[:n] != ab[:n])[0][:5]}"
    for m in sa:
        assert np.array_equal(sa[m], sb[m]), f"{what}: {m}: {sa[m]} vs {sb[m]}"
    for m in ea:
        assert ea[m].shape[0] == eb[m].shape[0], f"{what}: {m}: {ea[m].shape[0]} vs {eb[m].shape[0]} events"
        if ea[m].shape[0]:
            w = ea[m].shape[1] - (4 if m == "nat_log_rb" else 0)
            assert np.array_equal(ea[m][:, :w], eb[m][:, :w]), f"{what}: {m} records differ"
    for m in ta:
        (ka, va_), (kb, vb_) = ta[m], tb[m]
        assert np.array_equal(ka, kb), f"{what}: {m}: key sets differ ({len(ka)} vs {len(kb)})"
        x, y = va_.copy(), vb_.copy()
        for off, ln in L.PADDING.get(m, ()):
            x[:, off:off + ln] = 0
            y[:, off:off + ln] = 0
        assert np.array_equal(x, y), f"{what}: {m}: values differ"


@pytest.mark.parametrize("name", ["pipeline_imix", "pipeline_64", "nat_cold_64", "nat_steady_64", "nat_ingress_64", "antispoof_64",
                                  "qos_64", "qos_egress_64", "pipeline_tc"])
def test_million_frames_against_reference(name):
    """Every bench workload at BASELINE scale (10 k subscribers / 1 M flows of config #3, 2^20 frames) against the
    reference oracle, bit for bit: verdicts, frame bytes, counters, event streams, table dumps.  pipeline_tc is
    pipeline_imix in the order of the reference's TC hooks (QoS before NAT)."""
    n = 1 << 20
    wl = W.BUILDERS["pipeline_imix" if name == "pipeline_tc" else name](n, 0, 1)
    if name == "pipeline_tc":
        wl.prog = "pipeline_tc"
    if wl.derive is not None:  # return traffic: derived from what the oracle's own prewarm translated
        from oracle.pyoracle import Oracle, available
        o = Oracle("reference" if available("reference") else "port")
        for m, k, v in wl.maps:
            assert o.update_batch(m, as_bytes(k), as_bytes(v)) == 0
        tr = []
        for prog, h, l in wl.prewarm:
            pa = o.arena(h.shape[0] * 64 + 64)
            pa[: h.shape[0] * 64] = h.reshape(-1)
            o.run(prog, pa, l.copy(), wl.now0 - 1, stride=64)
            tr.append(np.array(pa[: h.shape[0] * 64]))
        wl.headers, wl.lens = wl.derive(tr)
        o.free_arenas()
    arena, off16, stride = _arena(wl)
    steps = 1 if name == "nat_cold_64" else 3
    ref = _oracle_run(wl, arena, off16, stride, steps)
    gpu = _gpu_run(wl, arena, off16, stride, steps, "device")
    _same(ref, gpu, f"{name}: reference oracle vs gpu (device-resident)")


@pytest.mark.parametrize("case", ["pipeline_up", "pipeline_tc", "qos", "qos_egress", "nat_cold", "nat_cold_exhaust", "pipeline_up_miss"])
def test_fat_subscribers_against_reference(case):
    """A handful of subscribers with thousands of frames each: every subscriber's run spans many tiles of the ordered
    phase, so its token bucket, port counter and flow creation travel along the chain of warps (kernels.cu: ChainRec)
    — what one GPU of an 8-GPU job sees, pushed further.  Bit for bit against the reference oracle."""
    n = 1 << 17
    if case in ("pipeline_up", "pipeline_tc", "pipeline_up_miss"):
        wl = W.pipeline(n, 0, 1, n_subs=12, flows_per_sub=64 if case != "pipeline_up_miss" else 700)
        if case == "pipeline_tc":
            wl.prog = "pipeline_tc"
        if case == "pipeline_up_miss":
            wl.prewarm = []  # nothing pre-created: the first batch creates 700 flows per subscriber along the chain
    elif case in ("qos", "qos_egress"):
        wl = W.qos(n, 0, 1, n_subs=7, egress=case == "qos_egress")
    else:
        # 1024-port blocks (AllocateNAT): 900 flows fit, 1500 exhaust the block in mid-run (drops + sequential code)
        wl = W.nat(n, 0, 1, n_subs=9, flows_per_sub=900 if case == "nat_cold" else 1500, cold=True)
    arena, off16, stride = _arena(wl)
    steps = 1 if case.startswith("nat_cold") else 3
    ref = _oracle_run(wl, arena, off16, stride, steps)
    gpu = _gpu_run(wl, arena, off16, stride, steps, "device")
    _same(ref, gpu, f"fat subscribers / {case}: reference oracle vs gpu")


def test_tc_staging_holds_only_records_written():
    """pipeline_tc runs nat44_egress after the token bucket, in the ordered phase, for every frame the bucket passed
    — session hits included.  Those hits log nothing and must not take nat_log_rb staging space: a staging buffer
    of 2^15 records (more than the 21 845 of the reference's 1 MiB ring) has to hold one batch of 2^16 frames that
    are nearly all hits, and the few hundred new flows near its end keep their SESSION_CREATE records."""
    n = 1 << 16
    wl = W.pipeline(n, 0, 1, n_subs=1000, flows_per_sub=8, imix=False)
    wl.prog = "pipeline_tc"
    for i, (m, k, v) in enumerate(wl.maps):
        if m == "qos_ingress":  # every bucket rate-limited but deep: every frame waits for it, and passes
            v = v.copy()
            v["rate_bps"], v["burst_bytes"] = 10**12, 1 << 30
            v["tokens"] = v["burst_bytes"]
            wl.maps[i] = (m, k, v)
    tail = np.arange(n - 512, n)
    tail = tail[np.isin(wl.headers[tail, 23], (6, 17))]
    wl.headers[tail, 35] ^= 0x5A  # new source ports: new flows, late in index order
    arena, off16, stride = _arena(wl)
    ref = _oracle_run(wl, arena, off16, stride, 1)
    created = int(ref[1]["nat_stats_map"][5]) - len(wl.prewarm[0][2])
    assert created >= 200, created
    gpu = _gpu_run(wl, arena, off16, stride, 1, "device", sizing=dict(W.sizing(wl), event_capacity=1 << 15))
    _same(ref, gpu, "pipeline_tc, 2^16 frames, 2^15 staging records: reference oracle vs gpu")


@pytest.mark.parametrize("case", ["pipeline_up", "pipeline_tc", "qos"])
def test_jumbo_lengths_against_reference(case):
    """The ordered phase carries a frame's length in the spare bits of its ordering key (DevBatch.kshift); lengths
    of 2046 bytes and more do not fit and are looked up instead.  A header ring (64-byte slots) whose len[] runs from
    64 to 9000 bytes, around the 2046 boundary in particular, against the reference oracle."""
    n = 1 << 16
    wl = W.qos(n, 0, 1, n_subs=300) if case == "qos" else W.pipeline(n, 0, 1, n_subs=300, imix=False)
    if case == "pipeline_tc":
        wl.prog = "pipeline_tc"
    pick = np.array([64, 128, 1518, 2044, 2045, 2046, 2047, 2048, 4000, 9000], np.uint32)
    wl.lens = pick[(S.splitmix64_array(0x7B0, n) % np.uint64(len(pick))).astype(np.int64)]
    arena, off16, stride = _arena(wl)
    assert off16 is None and stride == 64
    ref = _oracle_run(wl, arena, off16, stride, 2)
    gpu = _gpu_run(wl, arena, off16, stride, 2, "device")
    _same(ref, gpu, f"jumbo lengths / {case}: reference oracle vs gpu")


@pytest.mark.parametrize("case", ["pipeline_up", "qos"])
def test_tables_too_large_for_packed_keys(case):
    """Subscriber tables beyond 2^21 slots: the ordering key needs more than KEY_BITS bits, the frame length no longer
    rides in it (DevBatch.kshift = 0, three radix passes) and the ordered phase looks lengths up.  Same results."""
    n = 1 << 16
    wl = W.qos(n, 0, 1, n_subs=500) if case == "qos" else W.pipeline(n, 0, 1, n_subs=500)
    arena, off16, stride = _arena(wl)
    ref = _oracle_run(wl, arena, off16, stride, 2)
    big = dict(W.sizing(wl), max_subscribers=(1 << 21) + 4096)  # capacity = 2 x that, rounded up: 2^23 slots
    gpu = _gpu_run(wl, arena, off16, stride, 2, "device", sizing=big)
    _same(ref, gpu, f"unpacked keys / {case}: reference oracle vs gpu")


@pytest.mark.parametrize("mode", ["device", "pinned"])
def test_dhcp_config5_against_reference(mode):
    """BASELINE config #5 at its full table size: 1 000 000 subscriber_pools entries (the map's max_entries), 99 % hits, 2^18 requests."""
    wl = W.dhcp(1 << 18, 0, 1, n_subs=1_000_000)  # the reference map holds MAX_SUBSCRIBERS = 1e6 (bpf/maps.h)
    arena, off16, stride = _arena(wl)
    ref = _oracle_run(wl, arena, off16, stride, 1)
    gpu = _gpu_run(wl, arena, off16, stride, 1, mode)
    _same(ref, gpu, f"dhcp (1 M subscriber_pools): reference oracle vs gpu ({mode})")


def test_full_size_feed_paths_agree_and_conserve():
    n = 1 << 22
    wl = W.pipeline(n, 0, 1, imix=True)
    arena, off16, stride = _arena(wl)
    dev = _gpu_run(wl, arena, off16, stride, 2, "device")
    pin = _gpu_run(wl, arena, off16, stride, 2, "pinned")  # 16 chunks of 2^18 frames through the 3-stage pipeline
    _same(dev, pin, "pipeline 2^22: device-resident vs pinned zero-copy")
    outs, stats, events, tables = dev
    v = np.concatenate([o[0] for o in outs])
    assert set(np.unique(v)) <= {0, 2}
    a, q, nat = stats["antispoof_stats"], stats["qos_stats_map"], stats["nat_stats_map"]
    total = 2 * n
    assert a[0] + a[1] == total                       # every frame was either allowed or dropped by antispoof
    assert a[1] == a[3] + a[4]                        # drops are IPv4 or IPv6 violations
    assert int((v == 2).sum()) == a[1] + q[1] + nat[3]  # dropped frames = antispoof + QoS + NAT drops
    assert q[0] + q[1] == a[0]                        # every frame antispoof let through met its token bucket
    assert events["spoof_events"].shape[0] == a[2]
    k, s = tables["nat_sessions"]
    ses = s.view(L.nat_session).reshape(-1)
    assert ses["packets_out"].sum() == nat[0]         # every SNATed frame (pre-warm included) is on exactly one session
    assert len(ses) == nat[5]
