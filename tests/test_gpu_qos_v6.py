"""IPv6 shaping (bng_qos_ipv6_enable, include/bng_b200.h): a dual-stack subscriber's IPv6 frames meet the token bucket
of their subscriber_ipv6 owner in qos_ingress_prog, qos_egress_prog, pipeline_up and pipeline_tc.

The oracle never sees subscriber_ipv6, so the expected results come from the oracle's programs run stage by stage.
The three programs of a pipeline share no map, so antispoof_ingress over the batch, then nat44_egress over its
survivors, then qos_ingress_prog over NAT's survivors keyed on the pre-NAT frame (pipeline_tc: antispoof, QoS, NAT)
is the oracle's own composition; a test below checks that on the golden scripts.  Shaping is then one substitution in
the QoS stage: an attributed IPv6 frame is replaced by its shadow, an IPv4 frame of the same len from the owner
(ingress) or to the owner (egress), and the frame's own bytes are what leaves the stage."""
import errno
import os
import re

import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import Dataplane
from bng_b200 import dataplane as D
from bng_b200 import layouts as L
from test_gpu_dualstack import (FEED_IDS, FEEDS, NO_DIR, DualBackend, _addr16, _et6, attributions, check_acct_idle,
                                expected_acct_idle, expected_li, inject, install, lpm_many, make_table, v6_frames)
from test_gpu_li import assert_records_equal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPED = ("qos_ingress_prog", "qos_egress_prog", "pipeline_up", "pipeline_tc")
EGRESS = ("qos_egress_prog",)
# the golden scripts that run one of the shaped programs
SCRIPTS = ("ipopts", "pipeline", "pipeline_noeim", "pipeline_tc", "pipeline_tc_noeim", "qos", "ticks")
CLOCKS = ("batch", "frame")


def _need(kind):
    if kind == "none":
        pytest.fail("no oracle library present on this box")


# ---------------------------------------------------------------------------
# the oracle, stage by stage
# ---------------------------------------------------------------------------
def shadow_owners(table, a, starts, have, idx, egress):
    """Owner of each frame of idx that the IPv6 rule attributes (-1: none): untagged 0x86DD, the 16 address bytes
    present, a covering prefix."""
    off = 38 if egress else 22
    ok = (have[idx] >= off + 16) & _et6(a, starts[idx])
    out = np.full(len(idx), -1, np.int64)
    if ok.any():
        out[ok] = lpm_many(table, _addr16(a, starts[idx[ok]], off))
    return out


class StagedOracle(harness.OracleBackend):
    """The oracle with the pipelines and the QoS programs run stage by stage over index lists of the batch; with a
    prefix table, the QoS stage shapes IPv6 frames through their shadows."""

    def __init__(self, kind, table=None):
        super().__init__(kind)
        self.table = table
        self.shadowed = 0  # IPv6 frames that met a bucket through a shadow

    def run(self, prog, arena, lens, now, off16, stride, prio, now_v=None):
        if prog not in SHAPED:
            return super().run(prog, arena, lens, now, off16, stride, prio, now_v)
        n = len(lens)
        starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(n, dtype=np.int64) * stride
        assert not (starts % 16).any(), "the stages address frames by 16-byte offsets"
        have = lens.astype(np.int64) if off16 is not None else np.minimum(lens.astype(np.int64), stride)
        oa = self.o.arena(len(arena) + 64)
        oa[:len(arena)] = arena
        oa[len(arena):] = 0

        def stage(p, idx, data):
            if len(idx) == 0:
                return np.zeros(0, np.uint8)
            l = lens[idx].copy()
            pr = None if prio is None else prio[idx].copy()
            nv = None if now_v is None else np.ascontiguousarray(now_v[idx])
            v = self.o.run(p, data, l, now, off16=(starts[idx] // 16).astype(np.uint32), priority=pr, now_v=nv)
            lens[idx] = l
            if pr is not None:
                prio[idx] = pr
            return v

        def qos(p, idx, src):
            """p over frames idx as they are in src, each attributed IPv6 frame through its shadow; src unchanged."""
            qa = self.o.arena(len(oa))
            qa[:] = src
            if self.table is not None and len(idx):
                eg = p in EGRESS
                own = shadow_owners(self.table, qa, starts, have, idx, eg)
                for i, o in zip(idx[own >= 0], own[own >= 0]):
                    s = int(starts[i])
                    qa[s + 12:s + 15] = (0x08, 0x00, 0x45)
                    at = s + (30 if eg else 26)
                    qa[at:at + 4] = np.frombuffer(int(o).to_bytes(4, "little"), np.uint8)
                self.shadowed += int((own >= 0).sum())
            return stage(p, idx, qa)

        verdict = np.zeros(n, np.uint8)
        everyone = np.arange(n)
        shot = L.TC_ACT_SHOT
        if prog in ("qos_ingress_prog", "qos_egress_prog"):
            verdict[:] = qos(prog, everyone, oa)
        else:
            v = stage("antispoof_ingress", everyone, oa)
            verdict[v == shot] = shot
            s1 = everyone[v != shot]
            if prog == "pipeline_up":
                pre = oa.copy()  # qos_ingress_prog keys on the frame as it entered NAT
                v = stage("nat44_egress", s1, oa)
                verdict[s1[v == shot]] = shot
                s2 = s1[v != shot]
                v = qos("qos_ingress_prog", s2, pre)
                verdict[s2[v == shot]] = shot
            else:
                v = qos("qos_ingress_prog", s1, oa)
                verdict[s1[v == shot]] = shot
                s2 = s1[v != shot]
                v = stage("nat44_egress", s2, oa)
                verdict[s2[v == shot]] = shot
        arena[:] = oa[:len(arena)]
        self.o.free_arenas()
        return verdict


def owners_of(script):
    """Subscriber addresses the script's map commands install in subscriber_nat, qos_ingress or qos_egress."""
    seen = []
    for st in script.steps:
        if st[0] == "update" and st[1] in ("subscriber_nat", "qos_ingress", "qos_egress"):
            for k in np.ascontiguousarray(st[2]).view("<u4").reshape(-1):
                if int(k) not in seen:
                    seen.append(int(k))
    return seen[:40]


def frame_clocks(script, seed=1):
    """The script with a clock per frame on every run that had one per batch: monotonic, spread over 0.5 ms, less
    than the gap between the golden scripts' batches, so that no clock goes backwards across batches."""
    r = np.random.default_rng(seed)
    out = harness.Script(script.name)
    for st in script.steps:
        if st[0] == "run" and st[8] is None:
            _, prog, arena, lens, now, off16, stride, prio, _ = st
            nv = (now + np.sort(r.integers(0, 500_000, len(lens)))).astype(np.uint64)
            st = ("run", prog, arena, lens, now, off16, stride, prio, nv)
        out.steps.append(st)
    return out


def shaped_attributions(script, want, kind, table):
    """attributions() of the IPv6 rule with shaping on: an IPv6 frame a shaped program drops (TC_ACT_SHOT) is its
    owner's too, unless antispoof dropped it."""
    runs, final = attributions(script, want, kind, table)
    out = []
    for r in runs:
        tag, prog, owner, v6, verdict, lens, clocks, dirset, lay, off16, spoof = r
        if owner is not None and prog in SHAPED:
            starts, have, a = lay
            idx = np.nonzero((verdict == L.TC_ACT_SHOT) & ~spoof)[0]
            own = shadow_owners(table, a, starts, have, idx, prog in EGRESS)
            owner, v6 = owner.copy(), v6.copy()
            owner[idx[own >= 0]] = own[own >= 0]
            v6[idx[own >= 0]] = True
        out.append((tag, prog, owner, v6, verdict, lens, clocks, dirset, lay, off16, spoof))
    return out, final


def bucket_drops6(runs):
    """IPv6 frames attributed with TC_ACT_SHOT: the bucket's IPv6 drops."""
    return sum(int((r[3] & (r[4] == L.TC_ACT_SHOT)).sum()) for r in runs if r[3] is not None)


class ShapingBackend(DualBackend):
    def __init__(self, table, targets, pinned, **opts):
        super().__init__(table, targets, pinned, **opts)
        self.dp.qos_ipv6_enable(True)


def check_shaped(script, table, targets, kind, pinned, what, **opts):
    """The GPU with shaping on against the staged oracle, then its records against the rule; returns the runs."""
    ora = StagedOracle(kind, table)
    want = harness.run_script(ora, script)
    be = ShapingBackend(table, targets, pinned, **opts)
    try:
        got = harness.run_script(be, script)
        harness.compare(want, got, f"{what}: staged {kind} oracle with shadows vs gpu with IPv6 shaping")
        runs, final = shaped_attributions(script, want, kind, table)
        acct, idle = expected_acct_idle(runs, final)
        check_acct_idle(be.dp, acct, idle, what)
        assert_records_equal(be.records, expected_li(runs, targets), what)
    finally:
        be.close()
    return runs, ora.shadowed


# ---------------------------------------------------------------------------
# 1. the golden scripts with IPv6 frames
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("script", SCRIPTS)
def test_staged_oracle_is_the_composition(script, ora_kind):
    """Without a table the stage-by-stage oracle gives exactly what the oracle's own programs give: this checks the
    checker.  CPU only."""
    _need(ora_kind)
    base = scenarios.ALL_SCRIPTS[script]()
    sc = inject(base, make_table(owners_of(base)))
    for s in (sc, frame_clocks(sc)):
        want = harness.run_script(harness.OracleBackend(ora_kind), s)
        got = harness.run_script(StagedOracle(ora_kind), s)
        harness.compare(want, got, f"{script}: oracle vs the oracle stage by stage")


@pytest.mark.gpu
@pytest.mark.parametrize("clock", CLOCKS)
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("script", SCRIPTS)
def test_golden_scripts_shaped(script, pinned, clock, ora_kind):
    _need(ora_kind)
    base = scenarios.ALL_SCRIPTS[script]()
    owners = owners_of(base)
    table = make_table(owners)
    sc = inject(base, table, share=0.4)
    if clock == "frame":
        sc = frame_clocks(sc)
    targets = {o: 100 + j for j, o in enumerate(owners[::3] + [NO_DIR])}
    check_shaped(sc, table, targets, ora_kind, pinned, f"{script} ({FEED_IDS[FEEDS.index(pinned)]}, {clock} clock)")


# ---------------------------------------------------------------------------
# 2. ordering under pressure: a few subscribers, thousands of frames each in one batch
# ---------------------------------------------------------------------------
def pressure_script(seed=4, n_sub=4, per_sub=3000, progs=SHAPED, frame_clock=True):
    """The pipeline script's maps, then for each program one batch in which n_sub subscribers each send (or, for
    qos_egress_prog, receive) per_sub frames, IPv4 and IPv6 interleaved, against buckets that hold about half of what
    they are offered.  Every subscriber has several prefixes, the second one a /60 inside the first one's /48; each
    subscriber's frames carry one MAC.  Returns (script, prefix table, subscriber addresses)."""
    r = np.random.default_rng(seed)
    base = scenarios.ALL_SCRIPTS["pipeline"]()
    sc = harness.Script("pressure")
    for st in base.steps:
        if st[0] in ("update", "delete"):
            sc.steps.append(st)
    run0 = next(st for st in base.steps if st[0] == "run" and st[5] is None)
    _, _, arena, lens, now, _, stride0, _, _ = run0
    a0 = np.asarray(arena, np.uint8).reshape(len(lens), stride0)
    src = a0[:, 26:30].copy().view("<u4").reshape(-1)
    et4 = (a0[:, 12] == 0x08) & (a0[:, 13] == 0x00)
    subs = [int(x) for x in dict.fromkeys(src[et4].tolist())][:n_sub]
    table = make_table(subs, seed=seed)
    stride = 256
    n = n_sub * per_sub
    who = r.permutation(np.repeat(np.arange(n_sub), per_sub))
    six = r.random(n) < 0.5
    up = np.zeros((n, stride), np.uint8)
    down = np.zeros((n, stride), np.uint8)
    l = r.integers(64, stride + 1, n).astype(np.uint32)
    for j, s in enumerate(subs):
        rows = np.nonzero((src == s) & et4)[0]
        rows = rows[(a0[rows, 6:12] == a0[rows[0], 6:12]).all(axis=1)]  # one MAC per subscriber
        mine = np.nonzero(who == j)[0]
        up[mine, :stride0] = a0[rows[r.integers(0, len(rows), len(mine))]]
        down[mine] = up[mine]
        down[mine, 30:34] = np.frombuffer(int(s).to_bytes(4, "little"), np.uint8)  # IPv4 downstream: to s
        tab = [t for t in table if t[2] == s] + ([t for t in table if t[0] == 60] if j == 0 else [])
        for i in mine[six[mine]]:
            pl, p, _ = tab[r.integers(0, len(tab))]
            bits = np.zeros(128, np.uint8)
            bits[:pl] = 1
            m = np.packbits(bits)
            addr = (p & m) | (r.integers(0, 256, 16, dtype=np.uint8) & ~m)
            for f in (up, down):
                f[i, 12:22] = (0x86, 0xDD, 0x60, 0, 0, 0, 0, 0, 17, 64)
                f[i, 22:38] = addr  # upstream: the source
                f[i, 38:54] = addr  # downstream: the destination
    offered = np.bincount(who, weights=l.astype(np.float64), minlength=n_sub)
    span = 10**9
    tb = np.zeros(n_sub, L.token_bucket)
    tb["rate_bps"] = (offered * 8 // 4).astype(np.uint64)  # a quarter of the offer refilled over the batch's second
    tb["burst_bytes"] = (offered // 4).astype(np.uint32)   # ... and a quarter in the bucket to start with
    tb["tokens"] = tb["burst_bytes"]
    tb["last_update"] = now
    tb["priority"] = np.arange(n_sub) + 1
    keys = np.array(subs, "<u4").view(np.uint8).reshape(-1, 4)
    sc.update("qos_ingress", keys, tb)
    sc.update("qos_egress", keys, tb)
    # antispoof lets every subscriber's IPv6 frames through (mode 3: violations pass) but the last one's
    macs = np.array([int.from_bytes(bytes(up[np.nonzero(who == j)[0][0], 6:12]), "big") for j in range(n_sub - 1)], "<u8")
    bind = np.zeros(n_sub - 1, L.subscriber_binding)
    bind["ipv4_addr"] = keys[:-1]
    bind["ipv4_valid"], bind["mode"] = 1, 3
    sc.update("subscriber_bindings", macs.view(np.uint8).reshape(-1, 8), bind)
    nv = (now + np.sort(r.integers(0, span, n))).astype(np.uint64)
    for k, prog in enumerate(progs):
        shift = k * 2 * span
        f = down if prog in EGRESS else up
        sc.run(prog, f.reshape(-1).copy(), l.copy(), now + shift + span, stride=stride,
               priority=np.zeros(n, np.uint32) if prog in EGRESS else None, now_v=nv + shift if frame_clock else None)
    return sc, table, subs


@pytest.mark.gpu
@pytest.mark.parametrize("frame_clock", [True, False], ids=["frame_clock", "batch_clock"])
def test_ordering_under_pressure(frame_clock, ora_kind):
    _need(ora_kind)
    sc, table, subs = pressure_script(frame_clock=frame_clock)
    targets = {subs[0]: 1, subs[1]: 2}
    runs, shadowed = check_shaped(sc, table, targets, ora_kind, False, "pressure", max_batch=1 << 15, event_capacity=1 << 17)
    assert shadowed > 15000, "too few IPv6 frames met a bucket"
    for r in runs:
        if r[2] is None or r[1] not in SHAPED:
            continue
        six = r[3]
        share = float((r[4][six] == L.TC_ACT_SHOT).mean())
        assert 0.2 < share < 0.9, f"{r[1]}: {share:.2f} of the IPv6 frames dropped; the buckets should drop about half"


@pytest.mark.gpu
def test_zero_copy_chunk_edges_shaped(ora_kind):
    """Batches across the zero-copy chunk size, half IPv6, per-frame clocks, on the pinned feed, for every program."""
    _need(ora_kind)
    base = scenarios.ALL_SCRIPTS["pipeline"]()
    owners = owners_of(base)
    table = make_table(owners)
    r = np.random.default_rng(11)
    sc = harness.Script("chunks")
    for st in base.steps:
        if st[0] in ("update", "delete"):
            sc.steps.append(st)
    keys = np.array(owners, "<u4").view(np.uint8).reshape(-1, 4)
    tb = np.zeros(len(owners), L.token_bucket)
    tb["rate_bps"], tb["burst_bytes"], tb["priority"] = 400_000, 20_000, 3
    tb["tokens"] = tb["burst_bytes"]
    sc.update("qos_ingress", keys, tb)
    sc.update("qos_egress", keys, tb)
    run0 = next(st for st in base.steps if st[0] == "run" and st[5] is None)
    _, _, arena, lens, now, _, stride, _, _ = run0
    arena = np.asarray(arena, np.uint8).reshape(-1)
    n0 = len(lens)
    for k, prog in enumerate(SHAPED):
        n = (1 << 18) - 1 if k % 2 == 0 else (1 << 18) + 33
        idx = r.integers(0, n0, n)
        a = arena.reshape(n0, stride)[idx]
        f, l6 = v6_frames(a[:, :12], table, r, n, stride)
        six = r.random(n) < 0.5
        a[six] = f[six]
        l = np.where(six, l6, lens[idx]).astype(np.uint32)
        nv = np.sort(r.integers(now, now + 10**9, n)).astype(np.uint64)
        sc.run(prog, a.reshape(-1), l, now, stride=stride, priority=np.zeros(n, np.uint32) if prog in EGRESS else None,
               now_v=nv)
        now += 2 * 10**9
    targets = {owners[0]: 7, owners[1]: 8}
    runs, shadowed = check_shaped(sc, table, targets, ora_kind, True, "chunk edges", max_batch=1 << 19,
                                  event_capacity=1 << 20)
    assert bucket_drops6(runs) > 1000, "too few IPv6 frames were dropped by a bucket"
    assert shadowed > 100000


# ---------------------------------------------------------------------------
# 4. off is today
# ---------------------------------------------------------------------------
def _observe(sc, table, targets, setup):
    be = DualBackend(table, targets, False, max_batch=1 << 15, event_capacity=1 << 17)
    try:
        setup(be.dp)
        be.dp.prof_enable(True)
        n0 = be.dp.launch_count
        got = harness.run_script(be, sc)
        return be.dp.launch_count - n0, set(be.dp.prof_read()), be.dp.acct_dump(), be.records, got
    finally:
        be.close()


def _same(x, y, what):
    (l0, k0, a0, r0, g0), (l1, k1, a1, r1, g1) = x, y
    assert l0 == l1, f"{what}: {l0} vs {l1} launches"
    assert k0 == k1, f"{what}: kernel names {sorted(k0 ^ k1)}"
    assert np.array_equal(a0[0], a1[0]) and np.array_equal(a0[1], a1[1]), f"{what}: accounting records"
    assert len(r0) == len(r1) and all(p[0] == q[0] and np.array_equal(p[1], q[1]) for p, q in zip(r0, r1)), f"{what}: records"
    harness.compare(g0, g1, what)


@pytest.mark.gpu
def test_off_is_today():
    sc, table, subs = pressure_script(per_sub=600)
    targets = {subs[0]: 1, subs[2]: 3}
    never = _observe(sc, table, targets, lambda dp: None)
    assert not any("v6>" in k and "classify" in k for k in never[1])

    def on_off(dp):
        dp.qos_ipv6_enable(True)
        dp.qos_ipv6_enable(False)

    _same(never, _observe(sc, table, targets, on_off), "on, then off")
    _same(never, _observe(sc, table, targets, lambda dp: dp.qos_ipv6_enable(False)), "off set explicitly")
    # an empty table: "on" launches what "off" launches
    empty_never = _observe(sc, [], targets, lambda dp: None)
    _same(empty_never, _observe(sc, [], targets, lambda dp: dp.qos_ipv6_enable(True)), "on with an empty table")
    # and a filled table with shaping on does launch the IPv6 instantiations, under their own names
    on = _observe(sc, table, targets, lambda dp: dp.qos_ipv6_enable(True))
    names = on[1]
    for k in ("k_qos_classify<v6>", "(k_pipe_classify<true, true, false, true, v6>)",
              "(k_pipe_classify<true, true, true, true, v6>)"):
        assert k in names, f"{k} not in {sorted(names)}"
    assert on[0] == never[0]


# ---------------------------------------------------------------------------
# 5. sharding: two contexts, frames steered to their owner's, against one context
# ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_sharded_union():
    sc, table, subs = pressure_script(per_sub=1500, n_sub=6)
    world = 2
    owner_shard = {}
    mac_of = {}
    for st in sc.steps:
        if st[0] != "run":
            continue
        _, prog, arena, lens, now, off16, stride, prio, nv = st
        a = np.asarray(arena).reshape(len(lens), stride)
        src = a[:, 26:30].copy().view("<u4").reshape(-1)
        for s in subs:
            i = np.nonzero((src == s) & (a[:, 12] == 0x08))[0][0]
            mac_of[s] = a[i, 6:12]
        break
    for s in subs:
        owner_shard[s] = D.shard_of_mac(int.from_bytes(bytes(mac_of[s]) + b"\0\0", "little"), world)
    ctxs = [Dataplane(max_subscribers=1 << 12, max_batch=1 << 15, event_capacity=1 << 17) for _ in range(world + 1)]
    try:
        for dp in ctxs:
            install(dp, table)
            dp.qos_ipv6_enable(True)
        for st in sc.steps:
            if st[0] in ("update", "delete"):
                for dp in ctxs:
                    (dp.update_batch(st[1], st[2], st[3], st[4]) if st[0] == "update" else dp.delete(st[1], st[2]))
                continue
            _, prog, arena, lens, now, off16, stride, prio, nv = st
            n = len(lens)
            a = np.asarray(arena).reshape(n, stride)
            if prog in EGRESS:  # downstream: by the owner of the destination (IPv6: its prefix's owner)
                dst = a[:, 30:34].copy().view("<u4").reshape(-1)
                own6 = lpm_many(table, a[:, 38:54])
                is6 = (a[:, 12] == 0x86) & (a[:, 13] == 0xDD)
                owner = np.where(is6, own6, dst)
                shard = np.array([owner_shard.get(int(o), 0) for o in owner])
            else:  # upstream: by MAC
                shard = np.array([D.shard_of_mac(int.from_bytes(bytes(m) + b"\0\0", "little"), world) for m in a[:, 6:12]])
            one = harness.GpuBackend(ctxs[world]).run(prog, a.reshape(-1).copy(), lens.copy(), now, None, stride,
                                                      None if prio is None else prio.copy(), nv)
            v = np.zeros(n, np.uint8)
            for k in range(world):
                idx = np.nonzero(shard == k)[0]
                if len(idx):
                    v[idx] = harness.GpuBackend(ctxs[k]).run(prog, a[idx].reshape(-1).copy(), lens[idx].copy(), now, None,
                                                             stride, None if prio is None else prio[idx].copy(),
                                                             None if nv is None else np.ascontiguousarray(nv[idx]))
            assert np.array_equal(v, one), f"{prog}: sharded verdicts differ"
            assert (v == L.TC_ACT_SHOT).any()
        for m in harness.STATS_MAPS:
            assert np.array_equal(ctxs[0].stats(m) + ctxs[1].stats(m), ctxs[world].stats(m)), m
        for m in ("qos_ingress", "qos_egress"):
            k1, v1 = ctxs[world].dump(m)
            parts = [ctxs[k].dump(m) for k in range(world)]
            for key, val in zip(k1, v1):
                s = int(key.view("<u4")[0])
                kk, vv = parts[owner_shard.get(s, 0)]  # (a bucket no frame reaches is the same on every shard)
                row = np.nonzero((kk == key).all(axis=1))[0][0]
                assert np.array_equal(vv[row], val), f"{m} {s:#010x}"
    finally:
        for dp in ctxs:
            dp.close()


# ---------------------------------------------------------------------------
# 6. the interface (no GPU)
# ---------------------------------------------------------------------------
def test_header_declares_the_call():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bng_b200.h")).read(), flags=re.S)
    assert re.search(r"int\s+bng_qos_ipv6_enable\s*\(\s*bng_ctx\s*\*\s*ctx\s*,\s*int\s+on\s*\)\s*;", src)


def test_binding_exposes_the_call():
    assert "bng_qos_ipv6_enable" in D.EXPORTED_SYMBOLS
    assert callable(Dataplane.qos_ipv6_enable)


def test_null_context_is_einval():
    lib = D.load_library()
    assert lib.bng_qos_ipv6_enable(None, 1) == -errno.EINVAL
    assert lib.bng_qos_ipv6_enable(None, 0) == -errno.EINVAL
