"""Per-subscriber idle detection (bng_idle_*): the GPU's records against the rule of include/bng_b200.h, restated here
from the oracle's inputs, outputs and verdicts, on the pageable, pinned and device feeds; the scan against the scan
rule restated in numpy; lifecycle, snapshots, deltas, launch counts and sharding.

The stamp rule: frames are attributed to an address exactly as accounting attributes them (tests/test_gpu_acct.py
restates that); a frame with verdict TC_ACT_OK raises the record's stamp of its direction to the frame's clock."""
import errno

import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import layouts as L
from bng_b200 import synth as S
from bng_b200 import workloads as W
from bng_b200.layouts import as_bytes
from test_gpu_acct import (ACCOUNTED, FEED_IDS, FEEDS, PIPES, SCRIPTS, UP, _addr_keys, _frame_fields, _pipeline_batch,
                           _pipeline_corpus, _qos_frames, _unlimited)
from test_oracle_fuzz import fuzz_script

pytestmark = pytest.mark.gpu

SEC = 10**9
NEVER = L.IDLE_NEVER


# ---------------------------------------------------------------------------
# the stamp rule, restated, checked after every batch
# ---------------------------------------------------------------------------
def _dirset(rep):
    return _addr_keys(rep.dump("subscriber_nat")[0]) | _addr_keys(rep.dump("qos_ingress")[0])


def _stamp(exp, script_step, prog, want, tag, rep, dirset):
    """Raises the expected stamps {address: [up or None, down or None]} by one batch of the oracle's run."""
    if script_step[0] == "run_from":
        d = script_step[2](want)
        arena, lens = d["arena"], d["lens"].astype(np.uint32)
        off16, stride, now, now_v = d.get("off16"), int(d.get("stride", 0)), int(d["now_ns"]), d.get("now_v")
    else:
        _, _, arena, lens, now, off16, stride, _, now_v = script_step
    if prog not in ACCOUNTED:
        return
    verdict = np.asarray(want[tag + "_verdict"])
    if prog in UP:
        dlen, et, addr = _frame_fields(arena, lens, off16, stride, 26)
        ok = (dlen >= 30) & et
    else:
        dlen, et, addr = _frame_fields(want[tag + "_frames"], lens, off16, stride, 30)
        ok = (dlen >= 34) & et
    if prog in PIPES:
        av = np.asarray(rep.run("antispoof_ingress", arena.copy(), lens.copy(), now, off16, stride, None))
        ok &= av != L.TC_ACT_SHOT
    clk = np.asarray(now_v, np.uint64) if now_v is not None else np.full(len(lens), now, np.uint64)
    d = 0 if prog in UP else 1
    for i in np.nonzero(ok & (verdict == L.TC_ACT_OK))[0]:
        a = int(addr[i])
        if a in dirset:
            r = exp.setdefault(a, [None, None])
            r[d] = int(clk[i]) if r[d] is None else max(r[d], int(clk[i]))


def check_stamps(dp, exp, dirset, what):
    addrs = np.array(sorted(dirset), dtype="<u4")
    recs, found = dp.idle_read(addrs)
    assert found.all(), f"{what}: {int((~found).sum())} addresses of the directory have no record"
    bad = []
    for a, r in zip(addrs.tolist(), recs):
        up, down = exp.get(a, [None, None])
        want = (up or 0, down or 0, 0, 0, (L.IDLE_UP if up is not None else 0) | (L.IDLE_DOWN if down is not None else 0))
        got = (int(r["up_ns"]), int(r["down_ns"]), int(r["since_ns"]), int(r["timeout_s"]), int(r["flags"]))
        if got != want:
            bad.append((a, got, want))
    assert not bad, f"{what}: {len(bad)} records differ, e.g. {bad[0][0]:#010x}: {bad[0][1]} vs {bad[0][2]}"


def run_stamped(script_fn, pinned, ora_kind, enable=ACCOUNTED, acct=(), **opts):
    """Runs the script on the GPU with idle detection on for `enable` (and accounting for `acct`), step by step against
    the oracle's results; after every batch the verdicts and frames must equal the oracle's and every record the
    restated stamps.  Returns the GPU backend (the caller closes it)."""
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    want = harness.run_script(harness.OracleBackend(ora_kind), script_fn())
    script = script_fn()
    be = harness.GpuBackend(pinned=pinned, **opts)
    rep = harness.OracleBackend(ora_kind)
    try:
        for p in enable:
            be.dp.idle_enable(p)
        for p in acct:
            be.dp.acct_enable(p)
        exp, dirset = {}, set()
        for si, st in enumerate(script.steps):
            tag = f"s{si:03d}"
            if st[0] in ("update", "delete"):
                if st[0] == "update":
                    be.update(st[1], st[2], st[3], st[4])
                    rep.update(st[1], st[2], st[3], st[4])
                else:
                    be.delete(st[1], st[2])
                    rep.delete(st[1], st[2])
                if st[1] in ("subscriber_nat", "qos_ingress"):
                    dirset = _dirset(rep)
                    for a in [a for a in exp if a not in dirset]:
                        del exp[a]  # the address lost both entries: its record ended
                continue
            if st[0] == "lookup":
                be.lookup(st[1], st[2])
                continue
            if st[0] == "drain":
                for m in harness.EVENT_MAPS:
                    be.drain(m)
                continue
            assert st[0] in ("run", "run_from"), st[0]
            if st[0] == "run_from":
                d = st[2](want)
                prog, arena, lens = st[1], d["arena"], d["lens"].astype(np.uint32)
                off16, stride, now, prio, now_v = d.get("off16"), int(d.get("stride", 0)), int(d["now_ns"]), d.get("priority"), d.get("now_v")
            else:
                _, prog, arena, lens, now, off16, stride, prio, now_v = st
            a, l = arena.copy(), lens.copy()
            p = None if prio is None else prio.copy()
            v = be.run(prog, a, l, now, off16, stride, p, now_v) if now_v is not None else be.run(prog, a, l, now, off16, stride, p)
            assert np.array_equal(np.asarray(v), want[tag + "_verdict"]), f"{script.name} {tag}: verdicts differ"
            assert np.array_equal(a, want[tag + "_frames"]), f"{script.name} {tag}: frames differ"
            _stamp(exp, st, prog, want, tag, rep, dirset)
            check_stamps(be.dp, exp, dirset, f"{script.name} {tag} ({prog})")
    except BaseException:
        be.close()
        raise
    finally:
        rep.close()
    return be


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("script", SCRIPTS)
def test_golden_scripts_stamps(script, pinned, ora_kind):
    run_stamped(scenarios.ALL_SCRIPTS[script], pinned, ora_kind).close()


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("seed", [11, 13])
@pytest.mark.parametrize("prog", ACCOUNTED)
def test_fuzz_corpora_stamps(prog, seed, pinned, ora_kind):
    run_stamped(lambda: fuzz_script(prog, seed), pinned, ora_kind).close()


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("n", [255, 256, 257, 1023, 1024, 1025, 2047, 2048, 2049])
def test_batch_sizes_at_tile_and_chunk_edges(n, pinned, ora_kind, monkeypatch):
    monkeypatch.setenv("BNG_ZC_CHUNK_LOG2", "10")  # zero-copy chunks of 1024 frames (read at bng_open)
    run_stamped(_pipeline_batch(n), pinned, ora_kind).close()


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("prog", ["qos_ingress_prog", "pipeline_up"])
def test_one_subscriber_per_frame_clock(prog, pinned, ora_kind):
    """2^16 frames of one subscriber in one batch, each with its own clock (other subscribers' frames around it in
    the pipeline): the group maximum of every warp, not its first frame's clock."""
    updates, frames, lens, now, stride = _pipeline_corpus()
    n = 1 << 16
    one = frames[np.nonzero(frames[:, 26:30].view("<u4").reshape(-1) == frames[0, 26:30].view("<u4")[0])[0][0]]
    big = np.tile(one, (n, 1))
    ln = np.full(n, 64, np.uint32) + (np.arange(n) % 7).astype(np.uint32)
    if prog == "pipeline_up":
        pick = np.random.Generator(np.random.PCG64(9)).integers(0, len(lens), n)
        mix = np.arange(n) % 5 == 0
        big[mix] = frames[pick[mix]]
    clocks = now + np.cumsum(np.random.Generator(np.random.PCG64(4)).integers(0, 3, n)).astype(np.uint64)

    def fn():
        sc = harness.Script(f"one_sub_clock_{prog}")
        sc.steps = list(updates)
        if prog == "qos_ingress_prog":
            sc.update("qos_ingress", one[26:30].reshape(1, 4), _unlimited(1))
        sc.run(prog, big.reshape(-1).copy(), ln.copy(), now, stride=stride, now_v=clocks)
        return sc
    run_stamped(fn, pinned, ora_kind, max_batch=n).close()


def test_dropped_frames_do_not_stamp():
    """A token bucket that passes the first frames of a batch and drops the rest: the stamp is the clock of the last
    frame that passed, not of the batch's last frame."""
    from bng_b200 import Dataplane
    ip = S.sub_ip(np.array([3]))
    with Dataplane(max_subscribers=64, max_batch=1 << 12) as dp:
        tb = np.zeros(1, L.token_bucket)
        tb["rate_bps"], tb["burst_bytes"], tb["tokens"], tb["last_update"] = 8000, 1000, 1000, 10**9
        assert dp.update_batch("qos_ingress", S.ip_bytes(ip), tb) == 0
        dp.idle_enable("qos_ingress_prog")
        a, l = _qos_frames(ip, 40)
        clocks = (10**9 + np.arange(40) * 10).astype(np.uint64)
        v = dp.run("qos_ingress_prog", a, l, 10**9, stride=64, now_v=clocks)
        passed = np.nonzero(v == L.TC_ACT_OK)[0]
        assert 0 < len(passed) < 40 and (v[passed[-1] + 1:] == L.TC_ACT_SHOT).all()
        r, found = dp.idle_read(S.ip_bytes(ip))
        assert found[0] and int(r[0]["up_ns"]) == int(clocks[passed[-1]]) and int(r[0]["flags"]) == L.IDLE_UP
        # a batch that is dropped entirely leaves the stamp where it was
        v = dp.run("qos_ingress_prog", a, l, 10**9 + 500, stride=64)
        assert (v == L.TC_ACT_SHOT).all()
        assert int(dp.idle_read(S.ip_bytes(ip))[0][0]["up_ns"]) == int(clocks[passed[-1]])


@pytest.mark.parametrize("prog", PIPES)
def test_antispoof_drops_do_not_stamp(prog, ora_kind):
    """Pipeline frames from subscribers' addresses with another subscriber's MAC: antispoof drops them, and the
    restated rule (checked by run_stamped) gives them no stamp although their source address has an entry."""
    updates, frames, lens, now, stride = _pipeline_corpus()
    forged = frames.copy()
    forged[:, 6:12] = np.roll(frames[:, 6:12], 7, axis=0)
    idx = np.arange(len(lens)) % 2 == 0
    batch = np.where(idx[:, None], forged, frames)

    def fn():
        sc = harness.Script(f"forged_{prog}")
        sc.steps = list(updates)
        sc.run(prog, batch.reshape(-1).copy(), lens.copy(), now, stride=stride)
        return sc
    rep = harness.OracleBackend(ora_kind)
    try:
        for st in updates:
            if st[0] == "update":
                rep.update(st[1], st[2], st[3], st[4])
        av = np.asarray(rep.run("antispoof_ingress", batch.reshape(-1).copy(), lens.copy(), now, None, stride, None))
        dirset = _dirset(rep)
    finally:
        rep.close()
    src = np.ascontiguousarray(batch[:, 26:30]).view("<u4").reshape(-1)
    assert sum(1 for i in np.nonzero(av == L.TC_ACT_SHOT)[0] if int(src[i]) in dirset) > 0, "no drop of an address with an entry"
    run_stamped(fn, False, ora_kind, enable=(prog,)).close()


# ---------------------------------------------------------------------------
# the scan
# ---------------------------------------------------------------------------
def scan_rule(recs, now, default_s, flags):
    """The records idle at `now` (bool[n]), from records read just before the scan."""
    f = recs["flags"].astype(np.int64)
    ref = recs["since_ns"].astype(np.uint64)
    if flags & L.IDLE_UP:
        ref = np.where((f & L.IDLE_UP) != 0, np.maximum(ref, recs["up_ns"]), ref)
    if flags & L.IDLE_DOWN:
        ref = np.where((f & L.IDLE_DOWN) != 0, np.maximum(ref, recs["down_ns"]), ref)
    t = np.where(recs["timeout_s"] == 0, np.uint64(default_s), recs["timeout_s"].astype(np.uint64))
    started = (f & L.IDLE_STARTED) != 0
    le = ref <= np.uint64(now)
    age = np.where(le, np.uint64(now) - np.where(le, ref, 0), np.uint64(0))
    return started & (t != NEVER) & le & (age > t * np.uint64(SEC))


def _scan_setup(dp, n, rng):
    ips = S.sub_ip(np.arange(n))
    keys = S.ip_bytes(ips)
    assert dp.update_batch("qos_ingress", keys, _unlimited(n)) == 0
    dp.idle_enable("qos_ingress_prog")
    dp.idle_enable("qos_egress_prog")
    return ips, keys


def _stamp_random(dp, ips, rng, t0, t1, frac=0.5, down=False):
    """One batch from a random half of the addresses with random clocks in [t0, t1), upstream or downstream."""
    pick = np.sort(rng.choice(len(ips), int(len(ips) * frac), replace=False))
    clocks = np.sort(rng.integers(t0, t1, len(pick)).astype(np.uint64))
    order = rng.permutation(len(pick))  # which address gets which (sorted) clock
    src = ips[pick[order]]
    n = len(src)
    lens = np.full(n, 64, np.uint32)
    if down:
        hdr = S.ipv4_headers(np.full(n, 0x020000000009, np.uint64), np.uint64(scenarios.GW_MAC), np.full(n, 0x08080808, np.uint32),
                             src, np.full(n, 17, np.uint32), np.full(n, 53, np.uint32), np.full(n, 4000, np.uint32), lens)
        v = dp.run("qos_egress_prog", hdr.reshape(-1).copy(), lens, int(t0), stride=64, now_v=clocks)
    else:
        hdr = S.ipv4_headers(np.full(n, 0x020000000001, np.uint64), np.uint64(scenarios.GW_MAC), src, np.full(n, 0x08080808, np.uint32),
                             np.full(n, 17, np.uint32), np.full(n, 4000, np.uint32), np.full(n, 53, np.uint32), lens)
        v = dp.run("qos_ingress_prog", hdr.reshape(-1).copy(), lens, int(t0), stride=64, now_v=clocks)
    assert (v == L.TC_ACT_OK).all()
    return src, clocks


def _check_scan(dp, keys, now, default_s, flags, cap=None):
    before, found = dp.idle_read(keys)
    assert found.all()
    addrs_all = np.ascontiguousarray(keys).view("<u4").reshape(-1)
    want = scan_rule(before, now, default_s, flags)
    got_a, got_r, n = dp.idle_scan(now, default_s, flags, cap=cap)
    assert n == int(want.sum()), (now, default_s, flags, n, int(want.sum()))
    assert len(got_a) == (n if cap is None else min(n, cap))
    idx = {int(a): i for i, a in enumerate(addrs_all)}
    for a, r in zip(got_a.tolist(), got_r):
        i = idx[a]
        assert want[i], f"{a:#010x} reported idle"
        assert r.tobytes() == before[i].tobytes()
    after, _ = dp.idle_read(keys)
    unstarted = (before["flags"] & L.IDLE_STARTED) == 0
    assert (after["since_ns"][unstarted] == now).all() and (after["flags"][unstarted] & L.IDLE_STARTED).all()
    assert after[~unstarted].tobytes() == before[~unstarted].tobytes()
    return n


def test_scan_rule():
    from bng_b200 import Dataplane
    rng = np.random.Generator(np.random.PCG64(21))
    n = 3000
    with Dataplane(max_subscribers=2 * n, max_batch=1 << 14) as dp:
        ips, keys = _scan_setup(dp, n, rng)
        t0 = 1000 * SEC
        # nobody is reported at the first scan, even with a zero timeout: it starts every record
        assert _check_scan(dp, keys, t0, 0, L.IDLE_UP | L.IDLE_DOWN) == 0
        assert dp.idle_scan(t0 + 1, 0, 3)[2] == n  # and one ns later everything that never sent is idle at timeout 0
        for k in range(4):
            _stamp_random(dp, ips, rng, t0 + k * 20 * SEC, t0 + (k + 1) * 20 * SEC, down=bool(k & 1))
        tos = rng.choice(np.array([0, 0, 5, 30, 60, 90, NEVER], np.uint32), n)
        assert dp.idle_timeout_set(keys, tos).all()
        # subscribers that arrive after the first scan: started by the next one
        late = S.ip_bytes(S.sub_ip(np.arange(n, n + 200)))
        assert dp.update_batch("qos_ingress", late, _unlimited(200)) == 0
        allk = np.concatenate([keys, late])
        for now in (t0 + 10 * SEC, t0 + 70 * SEC, t0 + 95 * SEC, t0 + 200 * SEC, t0 + 10**6 * SEC):
            for default_s in (0, 45, NEVER):
                for flags in (L.IDLE_UP, L.IDLE_DOWN, L.IDLE_UP | L.IDLE_DOWN):
                    _check_scan(dp, allk, now, default_s, flags)
        # a stamp later than now: never idle; reported records can be capped, the count stays
        _stamp_random(dp, ips, rng, t0 + 10**7 * SEC, t0 + 10**7 * SEC + 5, frac=0.3)
        total = _check_scan(dp, allk, t0 + 10**6 * SEC, 1, 3)
        assert total > 10
        _check_scan(dp, allk, t0 + 10**6 * SEC, 1, 3, cap=7)
        _check_scan(dp, allk, t0 + 10**6 * SEC, 1, 3, cap=0)
        # the boundary: exactly timeout seconds is not idle (">")
        one = keys[:1]
        r, _ = dp.idle_read(one)
        ref = max(int(r[0]["since_ns"]), int(r[0]["up_ns"]), int(r[0]["down_ns"]))
        assert dp.idle_timeout_set(one, [7]).all()
        a, _, _ = dp.idle_scan(ref + 7 * SEC, NEVER, 3)
        assert int(np.ascontiguousarray(one).view("<u4").reshape(-1)[0]) not in set(a.tolist())
        a, _, _ = dp.idle_scan(ref + 7 * SEC + 1, NEVER, 3)
        assert int(np.ascontiguousarray(one).view("<u4").reshape(-1)[0]) in set(a.tolist())


def test_timeout_set_last_value_wins_and_enoent():
    from bng_b200 import Dataplane
    with Dataplane(max_subscribers=1024, max_batch=1 << 10) as dp:
        keys = S.ip_bytes(S.sub_ip(np.arange(100)))
        assert dp.update_batch("qos_ingress", keys[:50], _unlimited(50)) == 0
        rng = np.random.Generator(np.random.PCG64(2))
        idx = rng.integers(0, 100, 5000)
        tos = rng.integers(1, 1 << 31, 5000).astype(np.uint32)
        found = dp.idle_timeout_set(keys[idx], tos)
        assert np.array_equal(found, idx < 50)
        last = {}
        for i, t in zip(idx.tolist(), tos.tolist()):
            last[i] = t
        r, f = dp.idle_read(keys)
        assert f[:50].all() and not f[50:].any()
        for i in range(50):
            assert int(r[i]["timeout_s"]) == last.get(i, 0), i
        assert (r[50:].view(np.uint8) == 0).all()
        # a second call, after the scratch of the first was put back
        assert dp.idle_timeout_set(keys[:3], [1, 2, 3]).all()
        assert dp.idle_read(keys[:3])[0]["timeout_s"].tolist() == [1, 2, 3]


# ---------------------------------------------------------------------------
# lifecycle
# ---------------------------------------------------------------------------
def _rec(dp, key):
    r, found = dp.idle_read(np.asarray(key).reshape(1, 4))
    return r[0] if found[0] else None


def test_lifecycle_of_a_record():
    from bng_b200 import Dataplane
    ips = S.sub_ip(np.arange(32))
    keys = S.ip_bytes(ips)
    with Dataplane(max_subscribers=32, max_batch=1 << 12) as dp:  # a 64-slot directory: slots are reused
        _, nat_v, _ = S.nat_blocks(32, ports_per_sub=8, port_lo=1024, port_hi=1024 + 8 * 8 - 1)
        assert dp.update_batch("qos_ingress", keys, _unlimited(32)) == 0
        assert dp.update_batch("subscriber_nat", keys[:16], nat_v[:16]) == 0
        dp.idle_enable("qos_ingress_prog")  # records exist from here: the ones of existing addresses start at zero
        r, found = dp.idle_read(keys)
        assert found.all() and (r.view(np.uint8) == 0).all()
        a, l = _qos_frames(ips, 2)
        dp.run("qos_ingress_prog", a, l, 10 * SEC, stride=64)
        assert dp.idle_timeout_set(keys[[0, 20]], [77, 88]).all()
        assert dp.idle_scan(11 * SEC, NEVER, 3)[2] == 0
        r0 = _rec(dp, keys[0])
        assert int(r0["up_ns"]) == 10 * SEC and int(r0["since_ns"]) == 11 * SEC and int(r0["timeout_s"]) == 77
        assert int(r0["flags"]) == L.IDLE_UP | L.IDLE_STARTED
        # one of the two entries goes, comes back: the same record
        assert dp.delete("qos_ingress", keys[0]) == 0
        assert _rec(dp, keys[0]).tobytes() == r0.tobytes()
        assert dp.update("qos_ingress", keys[0], _unlimited(1)) == 0
        assert _rec(dp, keys[0]).tobytes() == r0.tobytes()
        # both go, the address comes back: a new record, timeout back to the default
        assert dp.delete("qos_ingress", keys[20]) == 0
        assert _rec(dp, keys[20]) is None
        assert not dp.idle_timeout_set(keys[20:21], [5]).any()  # -ENOENT
        assert dp.update("qos_ingress", keys[20], _unlimited(1)) == 0
        assert _rec(dp, keys[20]).tobytes() == bytes(32)
        # bng_map_clear, and tombstoned slots claimed by other addresses
        assert dp.clear("qos_ingress") == 0 and dp.clear("subscriber_nat") == 0
        others = S.ip_bytes(S.sub_ip(np.arange(100, 132)))
        assert dp.update_batch("qos_ingress", others, _unlimited(32)) == 0
        r, found = dp.idle_read(others)
        assert found.all() and (r.view(np.uint8) == 0).all()
        # staged upserts are applied before a read, a timeout_set and a scan
        assert dp.delete("qos_ingress", others[0]) == 0
        staged = S.ip_bytes(S.sub_ip(np.array([200])))
        assert dp.update_staged("qos_ingress", staged[0], _unlimited(1)) == 0
        assert dp.idle_timeout_set(staged, [9]).all()
        assert dp.idle_read(staged)[1].all()


def test_sweep_eviction_rebuild_and_flush_keep_records():
    from bng_b200 import Dataplane
    n_subs = 4
    with Dataplane(max_subscribers=64, max_nat_sessions=64, max_eim_mappings=64, max_batch=1 << 12) as dp:
        sc = harness.Script("setup")
        scenarios.nat_maps(sc, n_subs, 64, 0x0E)
        for st in sc.steps:
            assert dp.update_batch(st[1], st[2], st[3]) == 0
        keys = S.ip_bytes(S.sub_ip(np.arange(n_subs)))
        dp.idle_enable("nat44_egress")
        assert dp.idle_timeout_set(keys, [300, 400, 500, 600]).all()
        last = np.zeros(n_subs, np.int64)
        r = np.random.Generator(np.random.PCG64(5))
        for step in range(12):
            n = 600
            sub = r.integers(0, n_subs, n)
            sport = (10000 + step * 1000 + r.integers(0, 900, n)).astype(np.uint32)
            lens = np.full(n, 64, np.uint32)
            hdr = S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), np.full(n, 0x08080808, np.uint32),
                                 np.full(n, 17, np.uint32), sport, np.full(n, 53, np.uint32), lens)
            clocks = ((step + 1) * SEC + np.arange(n)).astype(np.uint64)
            v = dp.run("nat44_egress", hdr.reshape(-1).copy(), lens, (step + 1) * SEC, stride=64, now_v=clocks)
            for s in range(n_subs):
                ok = np.nonzero((sub == s) & (v == 0))[0]
                if len(ok):
                    last[s] = max(last[s], int(clocks[ok[-1]]))
            if step == 5:
                dp.sweep(10**13)
            if step == 8:
                dp.nat_flush(keys[:2], 9 * SEC)
        assert dp.lru_evictions > 0 and dp.table_rebuilds > 0
        recs, found = dp.idle_read(keys)
        assert found.all()
        assert recs["up_ns"].astype(np.int64).tolist() == last.tolist() and (last > 0).all()
        assert recs["timeout_s"].tolist() == [300, 400, 500, 600]


# ---------------------------------------------------------------------------
# independence from accounting, launch counts, errors
# ---------------------------------------------------------------------------
def test_accounting_records_unchanged(ora_kind):
    from test_gpu_acct import _as_dict, run_accounted
    be, _ = run_accounted(scenarios.ALL_SCRIPTS["pipeline"], False, ora_kind)
    try:
        alone = _as_dict(*be.dp.acct_dump())
    finally:
        be.close()
    be = run_stamped(scenarios.ALL_SCRIPTS["pipeline"], False, ora_kind, acct=ACCOUNTED)
    try:
        both = _as_dict(*be.dp.acct_dump())
    finally:
        be.close()
    assert any(sum(r) for r in alone.values()) and both == alone


def _launches(acct, idle, disable_after=False):
    from bng_b200 import Dataplane
    updates, frames, lens, now, stride = _pipeline_corpus()
    with Dataplane(max_subscribers=1 << 12, max_nat_sessions=1 << 14, max_eim_mappings=1 << 14, max_batch=1 << 12) as dp:
        for st in updates:
            if st[0] == "update":
                dp.update_batch(st[1], st[2], st[3], st[4])
        out = []
        for prog in ACCOUNTED:
            if acct:
                dp.acct_enable(prog)
            if idle:
                dp.idle_enable(prog)
                if disable_after:
                    dp.idle_enable(prog, False)
            c0 = dp.launch_count
            dp.run(prog, frames.reshape(-1).copy(), lens.copy(), now, stride=stride)
            out.append(dp.launch_count - c0)
        return out


def test_launch_counts():
    base, acct = _launches(False, False), _launches(True, False)
    assert _launches(False, True, disable_after=True) == base  # records allocated, nothing enabled: today's launches
    assert _launches(False, True) == acct  # idle alone: the accounting pass, and nothing more
    assert _launches(True, True) == acct  # both: still one pass
    assert all(a == b + 1 for a, b in zip(acct, base))


def test_error_codes():
    from bng_b200 import BngError, Dataplane
    with Dataplane(max_subscribers=1 << 10, max_batch=1 << 10) as dp:
        assert dp.idle_scan(10 * SEC)[2] == 0  # no records yet: nobody
        r, found = dp.idle_read(S.ip_bytes(S.sub_ip(np.arange(2))))
        assert not found.any() and (r.view(np.uint8) == 0).all()
        for p in ("antispoof_ingress", "nat44_hairpin_xdp", "dhcp_fastpath_prog"):
            with pytest.raises(BngError) as e:
                dp.idle_enable(p)
            assert e.value.errno == errno.EOPNOTSUPP
        for p in (-1, 9, 1 << 20):
            with pytest.raises(BngError) as e:
                dp.idle_enable(p)
            assert e.value.errno == errno.EINVAL
        for flags in (0, 4, 8, 3 | 16):
            with pytest.raises(BngError) as e:
                dp.idle_scan(10 * SEC, 0, flags)
            assert e.value.errno == errno.EINVAL
        lib, h = dp.lib, dp.h
        assert lib.bng_idle_scan(h, 0, 0, 3, None, None, 1) == -errno.EINVAL
        assert lib.bng_idle_scan(h, 0, 0, 3, None, None, 0) == 0
        assert lib.bng_idle_scan(None, 0, 0, 3, None, None, 0) == -errno.EINVAL
        assert lib.bng_idle_read(h, None, 1, None, None) == -errno.EINVAL
        assert lib.bng_idle_read(h, None, 0, None, None) == 0
        assert lib.bng_idle_timeout_set(h, None, None, 1, None) == -errno.EINVAL
        assert lib.bng_idle_timeout_set(h, None, None, 0, None) == 0
        assert lib.bng_idle_enable(None, 2, 1) == -errno.EINVAL
        dp.idle_enable("pipeline_up", False)  # disabling what was never enabled


# ---------------------------------------------------------------------------
# snapshot / restore, deltas
# ---------------------------------------------------------------------------
def _qos_ctx(n, timeouts=None, **opts):
    from bng_b200 import Dataplane
    dp = Dataplane(max_subscribers=opts.pop("max_subscribers", 1 << 12), max_batch=1 << 12, **opts)
    keys = S.ip_bytes(S.sub_ip(np.arange(n)))
    assert dp.update_batch("qos_ingress", keys, _unlimited(n)) == 0
    dp.idle_enable("qos_ingress_prog")
    if timeouts is not None:
        assert dp.idle_timeout_set(keys, timeouts).all()
    return dp, keys


def _stamp_all(dp, keys, now):
    ips = np.ascontiguousarray(keys).view(">u4").reshape(-1).astype(np.uint32)  # key bytes are the wire order
    a, l = _qos_frames(ips, 1)
    assert (dp.run("qos_ingress_prog", a, l, now, stride=64) == 0).all()
    r, found = dp.idle_read(keys)
    assert found.all() and (r["up_ns"] == now).all() and (r["flags"] & L.IDLE_UP).all()


def _assert_restarted(dp, keys, timeouts):
    r, found = dp.idle_read(keys)
    assert found.all()
    assert r["timeout_s"].tolist() == list(np.asarray(timeouts, np.uint32).tolist())
    assert (r["flags"] == 0).all() and (r["up_ns"] == 0).all() and (r["down_ns"] == 0).all() and (r["since_ns"] == 0).all()


def test_snapshot_carries_timeouts_and_restarts_clocks():
    from bng_b200 import Dataplane
    n = 300
    tos = np.random.Generator(np.random.PCG64(3)).choice(np.array([0, 10, 3600, NEVER], np.uint32), n)
    dp, keys = _qos_ctx(n, tos)
    try:
        _stamp_all(dp, keys, 50 * SEC)
        dp.idle_scan(60 * SEC)
        blob = dp.snapshot()
        assert b"subscriber_idle" in blob
        with Dataplane(max_subscribers=1 << 11, max_batch=1 << 12) as other:
            other.restore(blob)  # another size; idle detection never enabled there
            _assert_restarted(other, keys, tos)
            assert other.idle_scan(61 * SEC)[2] == 0  # restarted: the first scan starts them
        stripped = harness.strip_section(blob, "subscriber_idle")
        with Dataplane(max_subscribers=1 << 12, max_batch=1 << 12) as other:
            other.idle_enable("qos_ingress_prog")
            other.restore(stripped)
            _assert_restarted(other, keys, np.zeros(n, np.uint32))
        dp.restore(stripped)  # over live records: defaults, clocks restarted
        _assert_restarted(dp, keys, np.zeros(n, np.uint32))
        dp.restore(blob)
        _assert_restarted(dp, keys, tos)
    finally:
        dp.close()
    # a context that never used idle detection writes no section
    from bng_b200 import Dataplane as D
    with D(max_subscribers=1 << 10, max_batch=1 << 10) as plain:
        assert plain.update_batch("qos_ingress", keys[:3], _unlimited(3)) == 0
        assert b"subscriber_idle" not in plain.snapshot()


def _idle_section(blob):
    return L.parse_delta(blob)[1].get("subscriber_idle")


def test_delta_replicates_timeouts_and_restarts_clocks():
    from bng_b200 import Dataplane
    n = 400
    rng = np.random.Generator(np.random.PCG64(8))
    tos = rng.choice(np.array([0, 10, 60, NEVER], np.uint32), n)
    act, keys = _qos_ctx(n, tos)
    sb = Dataplane(max_subscribers=1 << 11, max_batch=1 << 12)
    try:
        act.delta_enable()
        blob = act.delta_export()
        sec = _idle_section(blob)
        assert sec is not None and sec[0] == 7 and len(sec[2]) == n and sec[3].shape[1] == 4
        assert sb.delta_apply(blob) == 0
        _assert_restarted(sb, keys, tos)
        # steady state: stamps and scans on the active send nothing
        _stamp_all(act, keys, 5 * SEC)
        act.idle_scan(6 * SEC)
        blob = act.delta_export()
        sec = _idle_section(blob)
        assert sec is not None and len(sec[1]) == 0 and len(sec[2]) == 0
        sb.idle_enable("qos_ingress_prog")
        _stamp_all(sb, keys, 5 * SEC)
        sb.idle_scan(6 * SEC)
        assert sb.delta_apply(blob) == 0
        _assert_restarted(sb, keys, tos)  # every apply restarts the standby's clocks
        # changed timeouts, a deleted subscriber, a new one
        ch = rng.choice(n, 50, replace=False)
        tos[ch] = rng.integers(1, 1000, 50).astype(np.uint32)
        assert act.idle_timeout_set(keys[ch], tos[ch]).all()
        assert act.delete("qos_ingress", keys[0]) == 0
        new = S.ip_bytes(S.sub_ip(np.array([n + 5])))
        assert act.update("qos_ingress", new[0], _unlimited(1)) == 0
        assert act.idle_timeout_set(new, [42]).all()
        blob = act.delta_export()
        sec = _idle_section(blob)
        assert len(sec[2]) == len(set(ch.tolist()) - {0}) + 1 and len(sec[1]) == 1
        assert sb.delta_apply(blob) == 0
        _assert_restarted(sb, keys[1:], tos[1:])
        _assert_restarted(sb, new, [42])
        assert not sb.idle_read(keys[:1])[1][0]
        # FULL: everything, and the standby's own timeouts are replaced
        assert sb.idle_timeout_set(keys[1:2], [12345]).all()
        blob = act.delta_export(full=True)
        assert len(_idle_section(blob)[2]) == n
        assert sb.delta_apply(blob) == 0
        _assert_restarted(sb, keys[1:], tos[1:])
    finally:
        act.close()
        sb.close()


def test_failover_reports_nobody_idle_at_takeover():
    """The active's subscribers went quiet long ago by the standby's clock; after the takeover the standby's first
    scan reports nobody, and one timeout later it reports those still quiet."""
    from bng_b200 import Dataplane
    n = 100
    act, keys = _qos_ctx(n, np.full(n, 30, np.uint32))
    sb = Dataplane(max_subscribers=1 << 11, max_batch=1 << 12)
    try:
        act.delta_enable()
        t = 100 * SEC
        _stamp_all(act, keys, t)
        act.idle_scan(t)
        for k in range(5):  # heartbeats
            t += 10 * SEC
            assert sb.delta_apply(act.delta_export()) == 0
        # the active dies at t; the standby takes over 1000 s later by its clock
        sb.idle_enable("qos_ingress_prog")
        take = t + 1000 * SEC
        assert sb.idle_scan(take)[2] == 0
        _stamp_all(sb, keys[: n // 2], take + 10 * SEC)
        a, _, found = sb.idle_scan(take + 31 * SEC)
        assert found == n - n // 2
        assert set(a.tolist()) == set(np.ascontiguousarray(keys[n // 2:]).view("<u4").reshape(-1).tolist())
    finally:
        act.close()
        sb.close()


# ---------------------------------------------------------------------------
# sharding
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
    clocks = (wl.now0 + np.arange(n) * 7).astype(np.uint64)

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
            dp.idle_enable("pipeline_up")
            mw = (warm_shard == rank) if world_ > 1 else np.ones(len(warm_h), bool)
            dp.run("nat44_egress", warm_h[mw].reshape(-1).copy(), warm_l[mw].copy(), wl.now0 - 1, stride=64)
            mine = np.nonzero(frame_shard == rank)[0] if world_ > 1 else np.arange(n)
            for s in range(steps):
                dp.run(wl.prog, wl.headers[mine].reshape(-1).copy(), wl.lens[mine].copy(), wl.now0 + s * wl.now_step, stride=64,
                       now_v=clocks[mine] + np.uint64(s * wl.now_step))
            keys = S.ip_bytes(S.sub_ip(sub))
            r, found = dp.idle_read(keys)
            return {int(a): (int(x["up_ns"]), int(x["flags"])) for a, x, f in
                    zip(np.ascontiguousarray(keys).view("<u4").reshape(-1), r, found) if f}
        finally:
            dp.close()

    whole = run(0, 1)
    assert sum(1 for v in whole.values() if v[1]) > 0
    seen = set()
    for rank in range(world):
        part = run(rank, world)
        for a, rec in part.items():
            assert ip_shard[np.array([a], "<u4").tobytes()] == rank, f"{a:#010x} has a record on shard {rank}"
            assert rec == whole[a], f"{a:#010x}: shard {rank} {rec} vs unsharded {whole[a]}"
        seen |= set(part)
    assert seen == set(whole)
