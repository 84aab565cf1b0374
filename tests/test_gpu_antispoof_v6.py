"""Antispoof by delegated prefix (bng_antispoof_ipv6_prefixes_enable, include/bng_b200.h): with the flag on,
antispoof_ingress (standalone and in pipeline_up and pipeline_tc) allows an IPv6 frame the reference would drop when
the longest subscriber_ipv6 prefix covering its source belongs to the binding of its source MAC.

The oracle never sees subscriber_ipv6, so the expected results come from the oracle run stage by stage
(test_gpu_qos_v6.StagedOracle) with one substitution in its antispoof stage: each frame the rule allows is handed to
the oracle with a non-IP ethertype, which the reference allows with exactly packets_allowed += 1 and no event.  The
frame's own bytes go on to the next stages, which pass IPv6 and non-IP frames alike (with IPv6 shaping on, the QoS
stage's own shadow applies).  Which frames the rule allows is decided from the oracle's subscriber_bindings and
antispoof_config at the moment the batch runs, and from the prefix table as the script's commands left it."""
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
from test_gpu_dualstack import (FEED_IDS, FEEDS, NO_DIR, DualBackend, _addr16, attributions, check_acct_idle,
                                expected_acct_idle, expected_li, install, lpm_many, make_table, mask)
from test_gpu_li import assert_records_equal
from test_gpu_qos_v6 import EGRESS, SHAPED, StagedOracle, frame_clocks, shadow_owners
from test_oracle_fuzz import mutate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RULED = ("antispoof_ingress", "pipeline_up", "pipeline_tc")
PIPES = ("pipeline_up", "pipeline_tc")
# the golden scripts that run one of the programs the rule changes
SCRIPTS = ("antispoof", "ipopts", "pipeline", "pipeline_noeim", "pipeline_tc", "pipeline_tc_noeim", "ticks")
CLOCKS = ("batch", "frame")
NON_IP = (0x88, 0xB5)  # IEEE local experimental ethertype: antispoof_ingress allows it with packets_allowed += 1


def _need(kind):
    if kind == "none":
        pytest.fail("no oracle library present on this box")


def mac_key(m):
    return int.from_bytes(bytes(m), "big")


# ---------------------------------------------------------------------------
# the rule, on the oracle's own maps
# ---------------------------------------------------------------------------
def rule_allows(a, starts, have, bindings, cfg, table):
    """Per frame: the rule allows it where the reference drops it.  bindings: {MAC key: subscriber_binding record},
    cfg: the antispoof_config record, table: [(prefixlen, addr, owner)]."""
    n = len(starts)
    out = np.zeros(n, bool)
    if not n or not table:
        return out
    cand = np.nonzero((have >= 54) & (a[starts + 12] == 0x86) & (a[starts + 13] == 0xDD))[0]
    if not len(cand):
        return out
    src = _addr16(a, starts[cand], 22)
    owner = lpm_many(table, src)
    for j, i in enumerate(cand):
        b = bindings.get(mac_key(a[starts[i] + 6:starts[i] + 12]))
        if b is None or not b["ipv4_valid"]:
            continue
        mode = int(b["mode"])
        if mode in (0, 3):  # disabled, log-only: the reference allows every frame
            continue
        if b["ipv6_valid"]:
            if np.array_equal(src[j], b["ipv6_addr"]):
                continue  # the exact match
        elif mode == 2:
            continue  # loose mode without an IPv6 binding
        out[i] = owner[j] == int(np.asarray(b["ipv4_addr"]).view("<u4")[0])
    return out


class _ShadowedAntispoof:
    """The oracle library with antispoof_ingress seeing the frames at `starts` with a non-IP ethertype; the bytes
    are put back as soon as it returns, so every later stage sees the frame itself."""

    def __init__(self, o):
        self._o = o
        self.starts = np.zeros(0, np.int64)

    def __getattr__(self, k):
        return getattr(self._o, k)

    def run(self, prog, data, lens, now, **kw):
        s = self.starts
        if prog != "antispoof_ingress" or not len(s):
            return self._o.run(prog, data, lens, now, **kw)
        keep = (data[s + 12].copy(), data[s + 13].copy())
        data[s + 12], data[s + 13] = NON_IP
        try:
            return self._o.run(prog, data, lens, now, **kw)
        finally:
            data[s + 12], data[s + 13] = keep


class RuleOracle(StagedOracle):
    """StagedOracle with the antispoof stage shadowed by the rule (prefixes=True; False: nothing is shadowed, the
    checker of the checker).  shape: IPv6 shaping on too (the QoS stage's own shadows).  subscriber_ipv6 commands
    update the table the rule reads."""

    def __init__(self, kind, table, prefixes=True, shape=False):
        self.rule_table = list(table)
        super().__init__(kind, self.rule_table if shape else None)
        self.prefixes = prefixes
        self.o = _ShadowedAntispoof(self.o)
        self.allowed = []  # per run: the frames the rule allowed (None: a program the rule does not touch)

    def update(self, m, k, v, flags):
        if m != "subscriber_ipv6":
            return super().update(m, k, v, flags)
        keys = np.ascontiguousarray(k).reshape(-1, L.bng_ipv6_prefix_key.itemsize).view(L.bng_ipv6_prefix_key).reshape(-1)
        vals = np.ascontiguousarray(v).reshape(-1, 4).view("<u4").reshape(-1)
        for key, val in zip(keys, vals):
            pl, p = int(key["prefixlen"]), mask(key["addr"], int(key["prefixlen"]))
            self.rule_table[:] = [t for t in self.rule_table if not (t[0] == pl and np.array_equal(mask(t[1], pl), p))]
            self.rule_table.append((pl, p, int(val)))
        return 0

    def delete(self, m, k):
        if m != "subscriber_ipv6":
            return super().delete(m, k)
        key = np.ascontiguousarray(k).reshape(-1)[:20].view(L.bng_ipv6_prefix_key)[0]
        pl, p = int(key["prefixlen"]), mask(key["addr"], int(key["prefixlen"]))
        before = len(self.rule_table)
        self.rule_table[:] = [t for t in self.rule_table if not (t[0] == pl and np.array_equal(mask(t[1], pl), p))]
        return 0 if len(self.rule_table) < before else -errno.ENOENT

    def run(self, prog, arena, lens, now, off16, stride, prio, now_v=None):
        self.o.starts = np.zeros(0, np.int64)
        if prog not in RULED:
            self.allowed.append(None)
            return super().run(prog, arena, lens, now, off16, stride, prio, now_v)
        n = len(lens)
        starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(n, dtype=np.int64) * stride
        have = lens.astype(np.int64) if off16 is not None else np.minimum(lens.astype(np.int64), stride)
        allow = np.zeros(n, bool)
        if self.prefixes:
            bk, bv = self.o.dump("subscriber_bindings")
            recs = np.ascontiguousarray(bv).view(L.subscriber_binding).reshape(-1)
            bindings = {int(x): r for x, r in zip(np.ascontiguousarray(bk).view("<u8").reshape(-1), recs)}
            _, cv = self.o.dump("antispoof_config")
            cfg = np.ascontiguousarray(cv).view(L.antispoof_config).reshape(-1)[0]
            a = np.concatenate([np.asarray(arena, np.uint8).reshape(-1), np.zeros(64, np.uint8)])
            allow = rule_allows(a, starts, have, bindings, cfg, self.rule_table)
        self.allowed.append(allow)
        self.o.starts = starts[allow]
        try:
            return super().run(prog, arena, lens, now, off16, stride, prio, now_v)
        finally:
            self.o.starts = np.zeros(0, np.int64)


def rule_attributions(script, want, kind, table, allowed, shape):
    """attributions() of the IPv6 rule, with the frames the rule allowed not counted as antispoof's drops; with
    shaping on, an IPv6 frame a bucket dropped is its owner's (test_gpu_qos_v6.shaped_attributions)."""
    runs, final = attributions(script, want, kind, table)
    assert len(runs) == len(allowed)
    out = []
    for r, allow in zip(runs, allowed):
        tag, prog, owner, v6, verdict, lens, clocks, dirset, lay, off16, spoof = r
        if owner is not None and allow is not None:
            spoof = spoof & ~allow
        if shape and owner is not None and prog in SHAPED:
            starts, have, a = lay
            idx = np.nonzero((verdict == L.TC_ACT_SHOT) & ~spoof)[0]
            own = shadow_owners(table, a, starts, have, idx, prog in EGRESS)
            owner, v6 = owner.copy(), v6.copy()
            owner[idx[own >= 0]] = own[own >= 0]
            v6[idx[own >= 0]] = True
        out.append((tag, prog, owner, v6, verdict, lens, clocks, dirset, lay, off16, spoof))
    return out, final


class PrefixBackend(DualBackend):
    def __init__(self, table, targets, pinned, shape=False, **opts):
        super().__init__(table, targets, pinned, **opts)
        self.dp.antispoof_ipv6_prefixes_enable(True)
        if shape:
            self.dp.qos_ipv6_enable(True)


def check_rule(script, table, targets, kind, pinned, what, shape=False, records=True, **opts):
    """The GPU with the flag on against the rule-shadowed staged oracle, then its accounting, idle and interception
    records against §18's rule; returns the frames the rule allowed."""
    ora = RuleOracle(kind, table, shape=shape)
    want = harness.run_script(ora, script)
    be = PrefixBackend(table, targets, pinned, shape=shape, **opts)
    try:
        got = harness.run_script(be, script)
        harness.compare(want, got, f"{what}: staged {kind} oracle with the rule's shadows vs gpu")
        if records:
            runs, final = rule_attributions(script, want, kind, table, ora.allowed, shape)
            acct, idle = expected_acct_idle(runs, final)
            check_acct_idle(be.dp, acct, idle, what)
            assert_records_equal(be.records, expected_li(runs, targets), what)
    finally:
        be.close()
    return sum(int(a.sum()) for a in ora.allowed if a is not None)


# ---------------------------------------------------------------------------
# the cases: bindings and frames around the rule
# ---------------------------------------------------------------------------
def _v4(k):
    return bytes((100, 127, k >> 8, k & 0xFF))


def case_bindings(n=16):
    """Synthetic subscribers 100.127.0.k behind MACs 02:a6:00:00:00:k: per-binding modes 0-3, some without
    ipv6_valid, some without ipv4_valid.  Returns (MAC keys u8[n, 8], subscriber_binding[n], owner u32 per k)."""
    macs = np.array([[0x02, 0xA6, 0, 0, 0, k] for k in range(n)], np.uint8)
    b = np.zeros(n, L.subscriber_binding)
    own = []
    for k in range(n):
        b[k]["ipv4_addr"] = np.frombuffer(_v4(k), np.uint8)
        b[k]["ipv4_valid"] = 0 if k % 8 == 7 else 1
        b[k]["ipv6_valid"] = 0 if k % 3 == 2 else 1
        b[k]["mode"] = k % 4
        own.append(int(np.frombuffer(_v4(k), "<u4")[0]))
    keys = np.array([mac_key(m) for m in macs], "<u8").view(np.uint8).reshape(-1, 8)
    return macs, b, keys, own


def case_table(owners):
    """make_table over the owners; each binding's ipv6_addr is its /128 (the exact match)."""
    return make_table(owners)


def _host(p, pl, r):
    m = mask(np.full(16, 0xFF, np.uint8), pl)
    return (p & m) | (r.integers(0, 256, 16, dtype=np.uint8) & ~m)


def case_frames(macs, owners, table, golden_macs, r, n, cap):
    """n IPv6 frames (u8[n, cap], lens) across the rule's cases: sources in the binding's own delegated prefix and
    /64 (other than its ipv6_addr), its exact ipv6_addr, another subscriber's prefix, the other subscriber's /60
    nested in the first one's /48, no covering prefix, link-local, the NO_DIR prefix; MACs of the synthetic
    bindings, of the golden batch and unbound ones; tagged frames and frames shorter than 54 bytes."""
    by_owner = {}
    for pl, p, o in table:
        by_owner.setdefault(o, []).append((pl, p))
    nested = [(pl, p) for pl, p, o in table if pl == 60]
    f = np.zeros((n, cap), np.uint8)
    lens = np.zeros(n, np.uint32)
    for i in range(n):
        who = r.integers(0, 10)
        if who < 7:
            k = int(r.integers(0, len(macs)))
            mac, mine = macs[k], owners[k]
        elif who < 9 and len(golden_macs):
            mac, mine = golden_macs[r.integers(0, len(golden_macs))][6:12], None
        else:
            mac, mine = np.array([0x02, 0xEE, 0, 0, r.integers(0, 256), r.integers(0, 256)], np.uint8), None
        f[i, 0:6] = (0x02, 0, 0, 0, 0, 0x01)
        f[i, 6:12] = mac
        c = r.integers(0, 20)
        if mine is not None and c < 8:  # its own /48 or /56, its /64
            pl, p = [x for x in by_owner[mine] if x[0] < 128][r.integers(0, 2)]
            src = _host(p, pl, r)
        elif mine is not None and c < 10:  # the exact /128
            src = [x for x in by_owner[mine] if x[0] == 128][0][1].copy()
        elif c < 12:  # another subscriber's prefix
            o = owners[r.integers(0, len(owners))]
            pl, p = by_owner[o][r.integers(0, len(by_owner[o]))]
            src = _host(p, pl, r)
        elif c < 14 and nested:  # the /60 that the second subscriber holds inside the first one's /48
            src = _host(nested[0][1], 60, r)
            if r.integers(0, 2):
                f[i, 6:12] = macs[0]
        elif c < 16:
            src = r.integers(0, 256, 16, dtype=np.uint8)
            src[0] = 0x2A  # no covering prefix
        elif c < 18:
            src = np.zeros(16, np.uint8)
            src[0], src[1] = 0xFE, 0x80
            src[8:] = r.integers(0, 256, 8, dtype=np.uint8)
        else:
            src = _host(by_owner[NO_DIR][0][1], 64, r)
        tagged = r.integers(0, 12) == 0
        o = 4 if tagged else 0
        if tagged:
            f[i, 12:16] = (0x81, 0x00, 0x00, 0x0A)
        f[i, 12 + o:14 + o] = (0x86, 0xDD)
        f[i, 14 + o] = 0x60
        f[i, 20 + o], f[i, 21 + o] = 17, 64
        if 38 + o <= cap:
            f[i, 22 + o:38 + o] = src
        if 54 + o <= cap:
            f[i, 38 + o:54 + o] = _host(table[0][1], 48, r)
        lens[i] = r.choice([14, 30, 37, 38, 53, 54]) if r.integers(0, 8) == 0 else r.integers(62, 200)
    return f, np.minimum(lens, cap).astype(np.uint32)


def golden_bindings(script):
    """(MAC key, ipv4 owner) of the script's own bindings with ipv4_valid."""
    out = []
    for st in script.steps:
        if st[0] == "update" and st[1] == "subscriber_bindings":
            ks = np.ascontiguousarray(st[2]).view("<u8").reshape(-1)
            vs = np.ascontiguousarray(st[3]).view(L.subscriber_binding).reshape(-1)
            for k, v in zip(ks, vs):
                if v["ipv4_valid"]:
                    out.append((int(k), int(np.asarray(v["ipv4_addr"]).view("<u4")[0])))
    return out


def rule_script(base, seed=3, share=0.4, configs=True):
    """The golden script with the case bindings installed first and IPv6 case frames appended to every run of
    antispoof_ingress, pipeline_up and pipeline_tc (runs a later run_from reads keep their shape, as in
    test_gpu_dualstack.inject).  configs: before each such run, antispoof_config cycles through every default_mode
    with log_violations on and off.  Returns (script, prefix table)."""
    r = np.random.default_rng(seed)
    macs, binds, keys, own = case_bindings()
    gold = golden_bindings(base)
    owners = own + [o for _, o in gold if o not in own][:8]
    table = case_table(owners)
    # the golden bindings' exact IPv6 addresses are left as they are; the case bindings' are their /128s
    for k in range(len(binds)):
        binds[k]["ipv6_addr"] = [t for t in table if t[2] == own[k] and t[0] == 128][0][1]
    out = harness.Script(base.name + "_as6")
    # (a run_from step names earlier steps by index: nothing is inserted before the last one)
    last_rf = max([i for i, st in enumerate(base.steps) if st[0] == "run_from"], default=-1)
    steps = list(base.steps)
    if not any(st[0] == "run" and st[1] in RULED for st in steps[last_rf + 1:]):
        # a copy of the first such run, its clocks a second after every clock of the script (a clock that went back
        # would meet sessions last seen in its future)
        _, prog, arena, lens, now, off16, stride, prio, now_v = next(st for st in steps if st[0] == "run" and st[1] in RULED)
        last = max(max(st[4], int(st[8].max()) if st[8] is not None and len(st[8]) else 0) for st in steps if st[0] == "run")
        shift = last + 10**9 - now
        steps.append(("run", prog, arena, lens, now + shift, off16, stride, prio,
                      None if now_v is None else (now_v + np.uint64(shift)).astype(np.uint64)))
    runs = 0
    for si, st in enumerate(steps):
        if si == last_rf + 1:
            out.update("subscriber_bindings", keys, binds)
        if st[0] != "run" or si <= last_rf or st[1] not in RULED:
            out.steps.append(st)
            continue
        _, prog, arena, lens, now, off16, stride, prio, now_v = st
        if configs:
            cfg = np.zeros(1, L.antispoof_config)
            cfg["default_mode"], cfg["log_violations"] = runs % 4, (runs // 4 + 1) % 2
            out.update("antispoof_config", np.zeros(1, "<u4"), cfg)
        runs += 1
        arena = np.asarray(arena, np.uint8).reshape(-1)
        n = len(lens)
        k = max(64, int(n * share))
        starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(n, dtype=np.int64) * stride
        gm = np.stack([arena[s:s + 12] for s in starts[: min(n, 256)]]) if n else np.zeros((0, 12), np.uint8)
        cap = stride if off16 is None else 128
        f, l6 = case_frames(macs, own, table, gm, r, k, cap)
        if off16 is None:
            arena2, off2 = np.concatenate([arena, f.reshape(-1)]), None
        else:
            end = (len(arena) + 15) // 16
            arena2 = np.concatenate([arena, np.zeros(end * 16 - len(arena), np.uint8), f.reshape(-1)])
            off2 = np.concatenate([off16, end + np.arange(k, dtype=np.uint32) * (cap // 16)]).astype(np.uint32)
        perm = r.permutation(n + k) if off16 is not None else None  # (variable layouts: IPv6 frames mixed in)
        lens2 = np.concatenate([lens, l6]).astype(np.uint32)
        prio2 = None if prio is None else np.concatenate([prio, np.zeros(k, np.uint32)])
        nv2 = None if now_v is None else np.concatenate([now_v, np.full(k, now_v[-1] if n else now, np.uint64)])
        if perm is not None and now_v is None:
            off2, lens2 = off2[perm], lens2[perm]
            prio2 = None if prio2 is None else prio2[perm]
        out.steps.append(("run", prog, arena2, lens2, now, off2, stride, prio2, nv2))
    return out, table


def _targets(table):
    owners = sorted({t[2] for t in table})
    return {o: 100 + j for j, o in enumerate(owners[::3] + [NO_DIR])}


# ---------------------------------------------------------------------------
# 1. the checker, and the golden scripts with the case frames
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("script", SCRIPTS)
def test_shadowed_oracle_without_shadows_is_the_oracle(script, ora_kind):
    """With nothing shadowed, the extended staged oracle gives exactly what the oracle's own antispoof_ingress and
    pipelines give; and the rule finds frames to allow in every case script.  CPU only."""
    _need(ora_kind)
    sc, table = rule_script(scenarios.ALL_SCRIPTS[script]())
    for s in (sc, frame_clocks(sc)):
        want = harness.run_script(harness.OracleBackend(ora_kind), s)
        ora = RuleOracle(ora_kind, table, prefixes=False)
        harness.compare(want, harness.run_script(ora, s), f"{script}: oracle vs the extended staged oracle, unshadowed")
    ora = RuleOracle(ora_kind, table)
    harness.run_script(ora, sc)
    assert sum(int(a.sum()) for a in ora.allowed if a is not None) > 0, "the rule allowed no frame"


def test_rule_cases():
    """The rule on hand-made frames: which of the cases it allows.  CPU only."""
    macs, binds, keys, own = case_bindings()
    table = case_table(own)
    for k in range(len(binds)):
        binds[k]["ipv6_addr"] = [t for t in table if t[2] == own[k] and t[0] == 128][0][1]
    bindings = {int(x): b for x, b in zip(keys.view("<u8").reshape(-1), binds)}
    cfg = np.zeros(1, L.antispoof_config)[0]
    r = np.random.default_rng(0)
    p48 = [t for t in table if t[2] == own[0] and t[0] == 48][0][1]
    p64 = [t for t in table if t[2] == own[1] and t[0] == 64][0][1]
    nested = [t for t in table if t[0] == 60][0][1]

    def one(k, src, length=90, et=(0x86, 0xDD)):
        a = np.zeros(192, np.uint8)
        a[6:12] = macs[k]
        a[12:14] = et
        a[22:38] = src
        return bool(rule_allows(a, np.array([0]), np.array([length]), bindings, cfg, table)[0])

    # binding 1: strict (mode 1), ipv4_valid and ipv6_valid
    assert one(1, _host(p64, 64, r))                       # its /64, not its ipv6_addr
    assert not one(1, binds[1]["ipv6_addr"])               # the exact match: the reference already allows it
    assert not one(1, _host(p48, 48, r))                   # subscriber 0's prefix
    assert not one(1, _host(p64, 64, r), length=53)        # short
    assert not one(1, _host(p64, 64, r), et=(0x81, 0x00))  # tagged
    assert not one(1, _host(p64, 64, r), et=(0x08, 0x00))  # IPv4
    # binding 0 is mode 0 (disabled); 4 is mode 0, 5 mode 1, 6 mode 2, 7 mode 3 without ipv4_valid
    assert not one(0, _host(p48, 48, r))
    q5 = [t for t in table if t[2] == own[5] and t[0] < 128]
    assert one(5, _host(q5[0][1], q5[0][0], r)) and one(5, _host(q5[1][1], q5[1][0], r))
    # loose mode (6: ipv6_valid) still needs the exact match, so its prefixes widen it
    q6 = [t for t in table if t[2] == own[6] and t[0] == 64][0][1]
    assert one(6, _host(q6, 64, r))
    q7 = [t for t in table if t[2] == own[7] and t[0] == 64][0][1]
    assert not one(7, _host(q7, 64, r))                    # log-only, and no ipv4_valid
    # the other subscriber's /60 nested in binding 0's /48 belongs to subscriber 1: binding 1 (strict) gets it
    assert one(1, _host(nested, 60, r))
    bindings[int(keys.view("<u8")[0, 0])]["mode"] = 1
    assert not one(0, _host(nested, 60, r)) and one(0, _host(p48, 48, r))
    # binding 2: loose (mode 2) without ipv6_valid: the reference allows every source
    q2 = [t for t in table if t[2] == own[2] and t[0] == 64][0][1]
    assert not one(2, _host(q2, 64, r))


@pytest.mark.gpu
@pytest.mark.parametrize("clock", CLOCKS)
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("script", SCRIPTS)
def test_golden_scripts_prefixes(script, pinned, clock, ora_kind):
    _need(ora_kind)
    sc, table = rule_script(scenarios.ALL_SCRIPTS[script]())
    if clock == "frame":
        sc = frame_clocks(sc)
    allowed = check_rule(sc, table, _targets(table), ora_kind, pinned, f"{script} ({FEED_IDS[FEEDS.index(pinned)]}, {clock} clock)")
    assert allowed > 0


@pytest.mark.gpu
@pytest.mark.parametrize("clock", CLOCKS)
@pytest.mark.parametrize("script", ("pipeline", "pipeline_tc", "ipopts", "ticks"))
def test_golden_scripts_prefixes_and_shaping(script, clock, ora_kind):
    """IPv6 shaping on too: the frames the rule lets in meet their owner's bucket (pipelines) as §19 shapes them."""
    _need(ora_kind)
    sc, table = rule_script(scenarios.ALL_SCRIPTS[script]())
    if clock == "frame":
        sc = frame_clocks(sc)
    check_rule(sc, table, _targets(table), ora_kind, False, f"{script} with shaping ({clock} clock)", shape=True)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [False, True], ids=["plain", "shaped"])
def test_zero_copy_chunk_edges(shape, ora_kind):
    """Batches across the zero-copy chunk size, per-frame clocks, on the pinned feed, for each program the rule
    changes."""
    _need(ora_kind)
    base = scenarios.ALL_SCRIPTS["pipeline"]()
    macs, binds, keys, own = case_bindings()
    table = case_table(own)
    for k in range(len(binds)):
        binds[k]["ipv6_addr"] = [t for t in table if t[2] == own[k] and t[0] == 128][0][1]
    r = np.random.default_rng(17)
    sc = harness.Script("chunks")
    sc.steps = [st for st in base.steps if st[0] in ("update", "delete")]
    sc.update("subscriber_bindings", keys, binds)
    tb = np.zeros(len(own), L.token_bucket)
    tb["rate_bps"], tb["burst_bytes"], tb["priority"] = 400_000, 20_000, 3
    tb["tokens"] = tb["burst_bytes"]
    sc.update("qos_ingress", np.array(own, "<u4").view(np.uint8).reshape(-1, 4), tb)
    run0 = next(st for st in base.steps if st[0] == "run" and st[5] is None)
    _, _, arena, lens, now, _, stride, _, _ = run0
    a0 = np.asarray(arena, np.uint8).reshape(len(lens), stride)
    for j, prog in enumerate(RULED):
        n = (1 << 18) - 1 if j % 2 == 0 else (1 << 18) + 33
        idx = r.integers(0, len(lens), n)
        a = a0[idx].copy()
        f, l6 = case_frames(macs, own, table, a0[:256, :12], r, n, stride)
        six = r.random(n) < 0.5
        a[six] = f[six]
        l = np.where(six, l6, lens[idx]).astype(np.uint32)
        nv = np.sort(r.integers(now, now + 10**9, n)).astype(np.uint64)
        sc.run(prog, a.reshape(-1), l, now, stride=stride, now_v=nv)
        now += 2 * 10**9
    allowed = check_rule(sc, table, {own[1]: 7, own[5]: 8}, ora_kind, True, "chunk edges", shape=shape,
                         max_batch=1 << 19, event_capacity=1 << 20)
    assert allowed > 20000


# ---------------------------------------------------------------------------
# 2. mutated corpora (the test_oracle_fuzz mutators), flag on
# ---------------------------------------------------------------------------
def fuzz_rule_script(prog, seed):
    base = scenarios.ALL_SCRIPTS["antispoof" if prog == "antispoof_ingress" else "pipeline"]()
    sc, table = rule_script(base, seed=seed, configs=False)
    out = harness.Script(f"fuzz_{prog}_{seed}")
    out.steps = [st for st in sc.steps if st[0] in ("update", "delete")]
    run = next(st for st in sc.steps if st[0] == "run" and st[1] in RULED and st[5] is None)
    _, _, arena, lens, now, _, stride, _, _ = run
    frames = np.asarray(arena, np.uint8).reshape(len(lens), stride)
    f, l = mutate(frames, lens, seed * 7919 + len(prog), stride)
    for mode in range(4):
        cfg = np.zeros(1, L.antispoof_config)
        cfg["default_mode"], cfg["log_violations"] = mode, mode % 2
        out.update("antispoof_config", np.zeros(1, "<u4"), cfg)
        out.run(prog, f.reshape(-1).copy(), l.copy(), now + 5 + mode * 10**9, stride=stride)
        f, l = f[::-1].copy(), l[::-1].copy()
    return out, table


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [11, 13, 17, 23])
@pytest.mark.parametrize("prog", RULED)
def test_mutated_frames_prefixes(prog, seed, ora_kind):
    _need(ora_kind)
    sc, table = fuzz_rule_script(prog, seed)
    check_rule(sc, table, {}, ora_kind, seed % 2 == 1, f"fuzz {prog} seed {seed}", records=False)


# ---------------------------------------------------------------------------
# 3. off is today
# ---------------------------------------------------------------------------
def _observe(sc, table, setup):
    be = DualBackend(table, {}, False, max_batch=1 << 15, event_capacity=1 << 17)
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
    harness.compare(g0, g1, what)


@pytest.mark.gpu
def test_off_is_today():
    sc, table = rule_script(scenarios.ALL_SCRIPTS["ticks"]())
    never = _observe(sc, table, lambda dp: None)
    assert not any("as6>" in k or "k_antispoof<v6>" in k for k in never[1])

    def on_off(dp):
        dp.antispoof_ipv6_prefixes_enable(True)
        dp.antispoof_ipv6_prefixes_enable(False)

    _same(never, _observe(sc, table, on_off), "on, then off")
    _same(never, _observe(sc, table, lambda dp: dp.antispoof_ipv6_prefixes_enable(False)), "off set explicitly")
    empty_never = _observe(sc, [], lambda dp: None)
    _same(empty_never, _observe(sc, [], lambda dp: dp.antispoof_ipv6_prefixes_enable(True)), "on with an empty table")
    on = _observe(sc, table, lambda dp: dp.antispoof_ipv6_prefixes_enable(True))
    for k in ("k_antispoof<v6>", "(k_pipe_classify<true, true, false, true, as6>)",
              "(k_pipe_classify<true, true, true, true, as6>)"):
        assert k in on[1], f"{k} not in {sorted(on[1])}"
    assert on[0] == never[0]
    assert not np.array_equal(on[4]["st_antispoof_stats"], never[4]["st_antispoof_stats"])

    def both(dp):
        dp.antispoof_ipv6_prefixes_enable(True)
        dp.qos_ipv6_enable(True)

    names = _observe(sc, table, both)[1]
    for k in ("(k_pipe_classify<true, true, false, true, v6, as6>)", "(k_pipe_classify<true, true, true, true, v6, as6>)"):
        assert k in names, f"{k} not in {sorted(names)}"


# ---------------------------------------------------------------------------
# 4. table and binding changes take effect at the next batch
# ---------------------------------------------------------------------------
def _pkey(pl, addr):
    k = np.zeros(1, L.bng_ipv6_prefix_key)
    k["prefixlen"], k["addr"] = pl, addr
    return k.view(np.uint8).reshape(1, -1)


@pytest.mark.gpu
@pytest.mark.parametrize("staged", [False, True], ids=["direct", "staged"])
def test_changes_take_effect_at_the_next_batch(staged, ora_kind):
    _need(ora_kind)
    macs, binds, keys, own = case_bindings(4)
    table = case_table(own)
    binds["mode"] = 1
    for k in range(4):
        binds[k]["ipv6_addr"] = [t for t in table if t[2] == own[k] and t[0] == 128][0][1]
    r = np.random.default_rng(5)
    sc = harness.Script("changes")
    sc.update("subscriber_bindings", keys, binds)
    cfg = np.zeros(1, L.antispoof_config)
    cfg["default_mode"], cfg["log_violations"] = 1, 1
    sc.update("antispoof_config", np.zeros(1, "<u4"), cfg)
    f, l = case_frames(macs, own, table, np.zeros((0, 12), np.uint8), r, 512, 128)
    p1 = [t for t in table if t[2] == own[1] and t[0] == 64][0]
    now = 10**9

    def batch(prog):
        nonlocal now
        sc.run(prog, f.reshape(-1).copy(), l.copy(), now, stride=128)
        now += 10**9

    for prog in RULED:
        batch(prog)
    sc.delete("subscriber_ipv6", _pkey(p1[0], p1[1]))  # subscriber 1's /64 goes: its hosts are dropped again
    for prog in RULED:
        batch(prog)
    sc.update("subscriber_ipv6", _pkey(p1[0], p1[1]), np.array([own[2]], "<u4").view(np.uint8).reshape(1, 4))
    for prog in RULED:
        batch(prog)  # ... and handed to subscriber 2: now its hosts are 2's
    b = binds.copy()
    b[1]["ipv4_valid"], b[3]["mode"] = 0, 3
    sc.update("subscriber_bindings", keys, b)
    for prog in RULED:
        batch(prog)

    class Staged(PrefixBackend):
        def update(self, m, k, v, flags):
            if staged and m == "subscriber_ipv6":
                return self.dp.update_staged(m, k, v)
            return super().update(m, k, v, flags)

    ora = RuleOracle(ora_kind, table)
    want = harness.run_script(ora, sc)
    be = Staged(table, {}, False)
    try:
        harness.compare(want, harness.run_script(be, sc), f"changes ({'staged' if staged else 'direct'})")
    finally:
        be.close()
    per = [int(a.sum()) for a in ora.allowed]
    assert per[0] > 0 and per[3] < per[0] and per[6] >= per[3] and per[9] < per[6], per


# ---------------------------------------------------------------------------
# 5. sharding: frames steered by source MAC, the union of the shards against one context
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
def test_sharded_union(world):
    """antispoof_stats and IPv6 verdicts of 2 and 8 contexts, maps on every context and frames steered by source
    MAC, against one context."""
    sc, table = rule_script(scenarios.ALL_SCRIPTS["pipeline"](), share=1.0)
    ctxs = [Dataplane(max_subscribers=1 << 12, max_batch=1 << 15, event_capacity=1 << 17) for _ in range(world + 1)]
    try:
        for dp in ctxs:
            install(dp, table)
            dp.antispoof_ipv6_prefixes_enable(True)
        for st in sc.steps:
            if st[0] in ("update", "delete"):
                for dp in ctxs:
                    (dp.update_batch(st[1], st[2], st[3], st[4]) if st[0] == "update" else dp.delete(st[1], st[2]))
                continue
            _, prog, arena, lens, now, off16, stride, prio, nv = st
            if prog not in RULED:
                continue
            n = len(lens)
            arena = np.asarray(arena, np.uint8)
            starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(n, dtype=np.int64) * stride
            shard = np.array([D.shard_of_mac(int.from_bytes(bytes(arena[s + 6:s + 12]) + b"\0\0", "little"), world)
                              for s in starts])
            one = harness.GpuBackend(ctxs[world]).run(prog, arena.copy(), lens.copy(), now, off16, stride,
                                                      None if prio is None else prio.copy(), nv)
            v = np.zeros(n, np.uint8)
            for k in range(world):
                idx = np.nonzero(shard == k)[0]
                if not len(idx):
                    continue
                if off16 is None:
                    a = arena.reshape(n, stride)[idx].reshape(-1).copy()
                    o = None
                else:
                    a, o = arena.copy(), np.ascontiguousarray(off16[idx])
                v[idx] = harness.GpuBackend(ctxs[k]).run(prog, a, lens[idx].copy(), now, o, stride,
                                                         None if prio is None else prio[idx].copy(),
                                                         None if nv is None else np.ascontiguousarray(nv[idx]))
            # antispoof is stateless, so an IPv6 frame's verdict is its shard's (NAT and QoS pass IPv6); an IPv4
            # frame's may differ where one subscriber's address is sent from several MACs and so from several shards
            six = (arena[starts + 12] == 0x86) & (arena[starts + 13] == 0xDD)
            assert np.array_equal(v[six], one[six]), f"{prog}: sharded IPv6 verdicts differ"
        st = [sum(c.stats("antispoof_stats") for c in ctxs[:world]), ctxs[world].stats("antispoof_stats")]
        assert np.array_equal(st[0], st[1])
        assert int(st[1][0]) > 0
    finally:
        for dp in ctxs:
            dp.close()


# ---------------------------------------------------------------------------
# 6. state transfer does not carry the flag
# ---------------------------------------------------------------------------
def _probe(dp, sc):
    be = harness.GpuBackend(dp)
    out = []
    for st in sc.steps:
        if st[0] == "run" and st[1] in RULED:
            _, prog, arena, lens, now, off16, stride, prio, nv = st
            out.append(be.run(prog, np.asarray(arena).copy(), lens.copy(), now, off16, stride,
                              None if prio is None else prio.copy(), nv))
    return out


def _setup_script():
    sc, table = rule_script(scenarios.ALL_SCRIPTS["pipeline"](), configs=False)
    cfg = np.zeros(1, L.antispoof_config)
    cfg["default_mode"], cfg["log_violations"] = 1, 1
    sc.steps.insert(1, ("update", "antispoof_config", np.zeros((1, 4), np.uint8), cfg.view(np.uint8).reshape(1, -1), 0))
    return sc, table


def _maps(dp, sc):
    for st in sc.steps:
        if st[0] == "update":
            dp.update_batch(st[1], st[2], st[3], st[4])


@pytest.mark.gpu
def test_snapshot_and_delta_do_not_carry_the_flag():
    sc, table = _setup_script()
    src = Dataplane(max_subscribers=1 << 12, max_batch=1 << 15, event_capacity=1 << 17)
    dst = Dataplane(max_subscribers=1 << 12, max_batch=1 << 15, event_capacity=1 << 17)
    sb = Dataplane(max_subscribers=1 << 12, max_batch=1 << 15, event_capacity=1 << 17)
    try:
        src.delta_enable(True)
        install(src, table)
        _maps(src, sc)
        src.antispoof_ipv6_prefixes_enable(True)
        blob = src.snapshot()
        sb.delta_apply(src.delta_export())
        dst.restore(blob)
        plain = Dataplane(max_subscribers=1 << 12, max_batch=1 << 15, event_capacity=1 << 17)
        try:
            install(plain, table)
            _maps(plain, sc)
            off = _probe(plain, sc)
        finally:
            plain.close()
        on = _probe(src, sc)
        six = _six(sc)
        same = lambda x, y: all(np.array_equal(p[s], q[s]) for p, q, s in zip(x, y, six))  # noqa: E731
        assert not same(on, off)
        for dp, what in ((dst, "restored"), (sb, "standby")):
            assert same(_probe(dp, sc), off), f"{what}: the flag came along"
            dp.antispoof_ipv6_prefixes_enable(True)
            assert same(_probe(dp, sc), on), f"{what}: with the flag set, the IPv6 verdicts differ from the source's"
    finally:
        for dp in (src, dst, sb):
            dp.close()


@pytest.mark.gpu
def test_hand_over_does_not_carry_the_flag():
    sc, table = _setup_script()
    owners = sorted({t[2] for t in table})
    src = Dataplane(max_subscribers=1 << 12, max_batch=1 << 15, event_capacity=1 << 17)
    dst = Dataplane(max_subscribers=1 << 12, max_batch=1 << 15, event_capacity=1 << 17)
    try:
        install(src, table)
        _maps(src, sc)
        for st in sc.steps:  # the destination holds the configuration; the subscribers come with the blob
            if st[0] == "update" and st[1] in ("antispoof_config",):
                dst.update_batch(st[1], st[2], st[3], st[4])
        src.antispoof_ipv6_prefixes_enable(True)
        before = _probe(src, sc)
        macs = np.concatenate([np.ascontiguousarray(st[2]).view("<u8").reshape(-1) for st in sc.steps
                               if st[0] == "update" and st[1] == "subscriber_bindings"])
        blob = src.sub_export(np.array(owners, "<u4"), macs=macs, detach=True)
        dst.sub_import(blob)
        got = _probe(dst, sc)
        assert any(not np.array_equal(g[s], b[s]) for g, b, s in zip(got, before, _six(sc))), \
            "the flag came with the subscribers"
        dst.antispoof_ipv6_prefixes_enable(True)
        src2 = Dataplane(max_subscribers=1 << 12, max_batch=1 << 15, event_capacity=1 << 17)
        try:
            install(src2, table)
            _maps(src2, sc)
            src2.antispoof_ipv6_prefixes_enable(True)
            want = _probe(src2, sc)
        finally:
            src2.close()
        got = _probe(dst, sc)
        for g, w, s in zip(got, want, _six(sc)):
            assert np.array_equal(g[s], w[s]), "the destination's IPv6 verdicts differ from the source's"
    finally:
        src.close()
        dst.close()


def _six(sc):
    return [np.nonzero(_is6(st))[0] for st in sc.steps if st[0] == "run" and st[1] in RULED]


def _is6(st):
    _, prog, arena, lens, now, off16, stride, prio, nv = st
    a = np.asarray(arena, np.uint8)
    starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(len(lens), dtype=np.int64) * stride
    return (a[starts + 12] == 0x86) & (a[starts + 13] == 0xDD)


# ---------------------------------------------------------------------------
# 7. the interface (no GPU)
# ---------------------------------------------------------------------------
def test_header_declares_the_call():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bng_b200.h")).read(), flags=re.S)
    assert re.search(r"int\s+bng_antispoof_ipv6_prefixes_enable\s*\(\s*bng_ctx\s*\*\s*ctx\s*,\s*int\s+on\s*\)\s*;", src)


def test_binding_exposes_the_call():
    assert "bng_antispoof_ipv6_prefixes_enable" in D.EXPORTED_SYMBOLS
    assert callable(Dataplane.antispoof_ipv6_prefixes_enable)


def test_null_context_is_einval():
    lib = D.load_library()
    assert lib.bng_antispoof_ipv6_prefixes_enable(None, 1) == -errno.EINVAL
    assert lib.bng_antispoof_ipv6_prefixes_enable(None, 0) == -errno.EINVAL
