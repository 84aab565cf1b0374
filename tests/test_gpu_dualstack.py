"""Dual-stack attribution (subscriber_ipv6, include/bng_b200.h): accounting, idle stamps and interception records of
IPv6 frames against the rule, restated here from the oracle's inputs, outputs and verdicts, the directory after each
replayed map command, and a Python longest-prefix match over the table.  The oracle never sees subscriber_ipv6: the
table lives on the GPU side and in this file.

The rule: an untagged Ethernet II frame with ethertype 0x86DD whose address bytes are present (source 22-37 upstream,
destination 38-53 downstream, as the frame leaves) belongs to the value of the longest prefix covering the address,
a subscriber IPv4 address; only a TC_ACT_OK frame is attributed.  From there the IPv4 rule applies unchanged."""
import errno

import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import BngError, Dataplane
from bng_b200 import dataplane as D
from bng_b200 import layouts as L
from test_gpu_acct import FIELDS, _addr_keys, _as_dict, _frame_fields
from test_gpu_li import _layout, _u32_at, got_records, assert_records_equal

pytestmark = pytest.mark.gpu

UP = ("nat44_egress", "qos_ingress_prog", "pipeline_up", "pipeline_tc")
DOWN = ("nat44_ingress", "qos_egress_prog")
PIPES = ("pipeline_up", "pipeline_tc")
ACCOUNTED = UP + DOWN
FEEDS = [False, True, "device"]
FEED_IDS = ["pageable", "pinned", "device"]
SCRIPTS = [s for s in sorted(scenarios.ALL_SCRIPTS) if s not in ("antispoof", "dhcp")]
NO_DIR = 0x0171A8C0  # 192.168.113.1: owns prefixes, never a directory entry


# ---------------------------------------------------------------------------
# the table and its longest-prefix match
# ---------------------------------------------------------------------------
def _net(i, hi=0x20, lo=0x01):
    """A /48 per i: 20hi:0d<lo>:<i>::/48."""
    a = np.zeros(16, np.uint8)
    a[0], a[1], a[2], a[3], a[4], a[5] = hi, 0x01, 0x0D, lo, (i >> 8) & 0xFF, i & 0xFF
    return a


def make_table(owners, seed=5):
    """[(prefixlen, addr u8[16], owner u32)] for a list of subscriber addresses: per subscriber a /128, a /64 and a
    delegated /56 or /48; nested prefixes of two subscribers; prefixes of an address without a directory entry."""
    r = np.random.default_rng(seed)
    t = []
    for j, o in enumerate(owners):
        base = _net(j)
        wan = base.copy()
        wan[6], wan[7] = 0xFF, 0x01
        host = wan.copy()
        host[8:] = r.integers(0, 256, 8, dtype=np.uint8)
        t.append((128, host, o))
        t.append((64, wan, o))
        t.append((56 if j % 2 else 48, base, o))
    if len(owners) >= 2:  # the second subscriber holds a /60 inside the first's /48: longest wins
        inner = _net(0)
        inner[6], inner[7] = 0x12, 0x30
        t.append((60, inner, owners[1]))
    t.append((64, _net(4000, lo=0x77), NO_DIR))
    return t


def mask(addr, pl):
    a = np.asarray(addr, np.uint8).copy()
    for j in range(16):
        keep = min(max(pl - 8 * j, 0), 8)
        a[j] &= (0xFF << (8 - keep)) & 0xFF
    return a


def lpm(table, addr, maxlen=128):
    best = None
    for pl, p, o in table:
        if pl <= maxlen and (best is None or pl > best[0]) and np.array_equal(mask(addr, pl), mask(p, pl)):
            best = (pl, o)
    return None if best is None else best[1]


def lpm_many(table, addrs):
    """lpm() of every row of u8[n, 16]: owner per row, -1 for none."""
    addrs = np.asarray(addrs, np.uint8).reshape(-1, 16)
    out = np.full(len(addrs), -1, np.int64)
    by_len = {}
    for pl, p, o in table:
        by_len.setdefault(pl, {})[mask(p, pl).tobytes()] = o
    for pl in sorted(by_len, reverse=True):
        m = mask(np.full(16, 0xFF, np.uint8), pl)
        rows = np.nonzero(out < 0)[0]
        masked = addrs[rows] & m
        d = by_len[pl]
        for i, row in zip(rows, masked):
            o = d.get(row.tobytes())
            if o is not None:
                out[i] = o
    return out


def dump_model(dp):
    keys, vals = dp.dump("subscriber_ipv6")
    return sorted((int(k.view("<u4")[0]), bytes(k[4:]), int(v.view("<u4")[0])) for k, v in zip(keys, vals))


def model_of(entries):
    return sorted((pl, bytes(mask(p, pl)), o) for pl, p, o in entries)


def install(dp, table):
    if not table:
        return
    keys = np.zeros(len(table), L.bng_ipv6_prefix_key)
    keys["prefixlen"] = [t[0] for t in table]
    keys["addr"] = np.stack([t[1] for t in table])
    assert dp.ipv6_prefixes_set(keys["addr"], keys["prefixlen"], np.array([t[2] for t in table], "<u4")) == 0


def sample_addrs(table, r, n):
    """Addresses inside the table's prefixes (host bits random), outside every prefix, and link-local."""
    out = []
    for _ in range(n):
        k = r.integers(0, 10)
        if k < 7:
            pl, p, _ = table[r.integers(0, len(table))]
            a = r.integers(0, 256, 16, dtype=np.uint8)
            m = mask(np.full(16, 0xFF, np.uint8), pl)
            out.append((p & m) | (a & ~m))
        elif k < 9:
            a = r.integers(0, 256, 16, dtype=np.uint8)
            a[0] = 0x2A  # 2a..::/8 holds no prefix
            out.append(a)
        else:
            a = np.zeros(16, np.uint8)
            a[0], a[1] = 0xFE, 0x80
            a[8:] = r.integers(0, 256, 8, dtype=np.uint8)
            out.append(a)
    return out


# ---------------------------------------------------------------------------
# IPv6 frames mixed into the golden scripts
# ---------------------------------------------------------------------------
def v6_frames(macs, table, r, n, cap):
    """n IPv6 frames (u8[n, cap], lens): UDP over IPv6, with short frames, VLAN-tagged ones, and both addresses drawn
    from the table; MACs taken from the batch so that antispoof sees bindings (and drops some sources)."""
    src, dst = sample_addrs(table, r, n), sample_addrs(table, r, n)
    f = np.zeros((n, cap), np.uint8)
    lens = np.zeros(n, np.uint32)
    for i in range(n):
        f[i, :12] = macs[r.integers(0, len(macs))]
        tagged = r.integers(0, 12) == 0
        o = 4 if tagged else 0
        if tagged:
            f[i, 12:16] = (0x81, 0x00, 0x00, 0x0A)
        f[i, 12 + o:14 + o] = (0x86, 0xDD)
        f[i, 14 + o] = 0x60
        f[i, 20 + o], f[i, 21 + o] = 17, 64
        f[i, 22 + o:38 + o] = src[i] if 38 + o <= cap else 0
        if 54 + o <= cap:
            f[i, 38 + o:54 + o] = dst[i]
        lens[i] = r.choice([30, 37, 38, 53, 54, 62, 90, 120]) if r.integers(0, 6) == 0 else r.integers(62, 200)
    return f, np.minimum(lens, cap).astype(np.uint32)  # a frame's storage holds its whole length


def inject(script, table, seed=3, share=0.3):
    """The script with IPv6 frames appended to its runs.  Runs whose results a later run_from step reads keep their
    shape (those steps stay as they are); when that leaves no run, an IPv6-carrying copy of the first run is appended."""
    r = np.random.default_rng(seed)
    out = harness.Script(script.name)
    last_rf = max([i for i, st in enumerate(script.steps) if st[0] == "run_from"], default=-1)
    steps = list(script.steps)
    if not any(st[0] == "run" for st in steps[last_rf + 1:]):
        steps.append(next(st for st in steps if st[0] == "run"))
    for si, st in enumerate(steps):
        if st[0] != "run" or si <= last_rf:
            out.steps.append(st)
            continue
        _, prog, arena, lens, now, off16, stride, prio, now_v = st
        arena = np.asarray(arena, np.uint8).reshape(-1)
        n = len(lens)
        k = max(1, int(n * share))
        starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(n, dtype=np.int64) * stride
        macs = np.stack([arena[s:s + 12] for s in starts[: min(n, 256)]]) if n else np.zeros((1, 12), np.uint8)
        cap = stride if off16 is None else 128
        f, l6 = v6_frames(macs, table, r, k, cap)
        if off16 is None:
            arena2 = np.concatenate([arena, f.reshape(-1)])
            off2 = None
        else:
            end = (len(arena) + 15) // 16
            arena2 = np.concatenate([arena, np.zeros(end * 16 - len(arena), np.uint8), f.reshape(-1)])
            off2 = np.concatenate([off16, end + np.arange(k, dtype=np.uint32) * (cap // 16)]).astype(np.uint32)
        lens2 = np.concatenate([lens, l6]).astype(np.uint32)
        prio2 = None if prio is None else np.concatenate([prio, np.zeros(k, np.uint32)])
        nv2 = None if now_v is None else np.concatenate([now_v, np.full(k, now_v[-1] if n else now, np.uint64)])
        out.steps.append(("run", prog, arena2, lens2, now, off2, stride, prio2, nv2))
    return out


def _et6(a, starts):
    return (a[starts + 12] == 0x86) & (a[starts + 13] == 0xDD)


def _addr16(a, starts, off):
    return np.stack([a[starts + off + k] for k in range(16)], axis=1)


def attributions(script, want, ora_kind, table):
    """Per run of the script: (tag, prog, owner per frame (-1: nobody), frame carried IPv6, verdict, lens, clocks, the
    directory when it ran, its input layout, its output layout, spoof drops)."""
    rep = harness.OracleBackend(ora_kind)
    runs = []
    try:
        for si, st in enumerate(script.steps):
            tag = f"s{si:03d}"
            if st[0] == "update":
                rep.update(st[1], st[2], st[3], st[4])
                continue
            if st[0] == "delete":
                rep.delete(st[1], st[2])
                continue
            if st[0] not in ("run", "run_from"):
                continue
            if st[0] == "run_from":
                d = st[2](want)
                prog, arena, lens = st[1], d["arena"], d["lens"].astype(np.uint32)
                off16, stride, now, now_v = d.get("off16"), int(d.get("stride", 0)), int(d["now_ns"]), d.get("now_v")
            else:
                _, prog, arena, lens, now, off16, stride, _, now_v = st
            dirset = _addr_keys(rep.dump("subscriber_nat")[0]) | _addr_keys(rep.dump("qos_ingress")[0])
            if prog not in ACCOUNTED:
                runs.append((tag, prog, None, None, None, lens, None, dirset, None, None, None))
                continue
            verdict = np.asarray(want[tag + "_verdict"])
            up = prog in UP
            src = arena if up else want[tag + "_frames"]
            dlen, et4, addr4 = _frame_fields(src, lens, off16, stride, 26 if up else 30)
            starts, have, a = _layout(src, lens, off16, stride)
            owner = np.full(len(lens), -1, np.int64)
            ok4 = (dlen >= (30 if up else 34)) & et4
            owner[ok4] = addr4[ok4]
            spoof = np.zeros(len(lens), bool)
            if prog in PIPES:
                a2, l2 = arena.copy(), lens.copy()
                spoof = np.asarray(rep.run("antispoof_ingress", a2, l2, now, off16, stride, None)) == L.TC_ACT_SHOT
                owner[spoof] = -1
            ok6 = np.nonzero((dlen >= (38 if up else 54)) & _et6(a, starts) & (verdict == L.TC_ACT_OK))[0]
            o6 = lpm_many(table, _addr16(a, starts[ok6], 22 if up else 38))
            v6 = np.zeros(len(lens), bool)
            owner[ok6[o6 >= 0]] = o6[o6 >= 0]
            v6[ok6[o6 >= 0]] = True
            clocks = np.asarray(now_v, np.uint64) if now_v is not None else np.full(len(lens), now, np.uint64)
            runs.append((tag, prog, owner, v6, verdict, lens, clocks, dirset, (starts, have, a), off16, spoof))
        final = _addr_keys(rep.dump("subscriber_nat")[0]) | _addr_keys(rep.dump("qos_ingress")[0])
    finally:
        rep.close()
    return runs, final


def expected_acct_idle(runs, final):
    recs, idle = {}, {}
    for tag, prog, owner, v6, verdict, lens, clocks, dirset, _, _, _ in runs:
        for a in [a for a in recs if a not in dirset]:
            del recs[a]
        for a in [a for a in idle if a not in dirset]:
            del idle[a]
        if owner is None:
            continue
        base = 0 if prog in UP else 4
        for i in np.nonzero((owner >= 0) & ((verdict == L.TC_ACT_OK) | (verdict == L.TC_ACT_SHOT)))[0]:
            a = int(owner[i])
            if a not in dirset:
                continue
            r = recs.setdefault(a, [0] * 8)
            j = base + (2 if verdict[i] == L.TC_ACT_SHOT else 0)
            r[j] += 1
            r[j + 1] += int(lens[i])
            if verdict[i] == L.TC_ACT_OK:
                s = idle.setdefault(a, [0, 0])
                k = 0 if prog in UP else 1
                s[k] = max(s[k], int(clocks[i]) + 1)
    return {a: recs.get(a, [0] * 8) for a in final}, {a: idle.get(a, [0, 0]) for a in final}


def expected_li(runs, targets, snaplen=1518):
    out, batch = [], 0
    for tag, prog, owner, v6, verdict, lens, clocks, _, lay, _, _ in runs:
        batch += 1
        if owner is None:
            continue
        starts, have, a = lay
        recs = []
        for i in np.nonzero(owner >= 0)[0]:
            o = int(owner[i])
            if o not in targets or verdict[i] not in (L.TC_ACT_OK, L.TC_ACT_SHOT):
                continue
            cl = int(min(int(lens[i]), int(have[i]), snaplen))
            h = dict(ts_ns=int(clocks[i]), batch=batch, frame=int(i), target_id=targets[o], addr=o, wire_len=int(lens[i]),
                     cap_len=cl, dir=L.LI_UPLINK if prog in UP else L.LI_DOWNLINK, verdict=int(verdict[i]),
                     prog=D.PROGRAMS.index(prog))
            recs.append((h, a[starts[i]:starts[i] + cl].copy()))
        out.extend(recs)
    return out


def script_owners(script):
    """The subscriber addresses the script's map commands install (subscriber_nat / qos_ingress keys)."""
    seen = []
    for st in script.steps:
        if st[0] == "update" and st[1] in ("subscriber_nat", "qos_ingress"):
            for k in np.ascontiguousarray(st[2]).view("<u4").reshape(-1):
                if int(k) not in seen:
                    seen.append(int(k))
    return seen[:40]


def check_acct_idle(dp, acct, idle, what):
    addrs, recs = dp.acct_dump()
    got = _as_dict(addrs, recs)
    assert set(got) == set(acct), f"{what}: the dump's addresses differ from the directory"
    bad = [a for a in acct if got[a] != acct[a]]
    assert not bad, f"{what}: {len(bad)} records differ, e.g. {bad[0]:#010x}: {got[bad[0]]} vs {acct[bad[0]]}"
    a = np.array(sorted(idle), "<u4")
    rec, found = dp.idle_read(a)
    assert found.all()
    for x, r in zip(a.tolist(), rec):
        want = idle[x]
        assert [int(r["up_ns"]) + (1 if r["flags"] & L.IDLE_UP else 0), int(r["down_ns"]) + (1 if r["flags"] & L.IDLE_DOWN else 0)] == want, \
            f"{what}: idle stamps of {x:#010x}: {r} vs {want}"


class DualBackend(harness.GpuBackend):
    """The GPU backend with subscriber_ipv6 filled before the script, accounting, idle stamps and interception on,
    draining the interception records after each run."""

    def __init__(self, table, targets, pinned, **opts):
        super().__init__(pinned=pinned, **opts)
        install(self.dp, table)
        for p in ACCOUNTED:
            self.dp.acct_enable(p)
            self.dp.idle_enable(p)
        self.dp.li_configure(0, 1 << 16)
        for a, t in targets.items():
            self.dp.li_target_set(a, t)
        self.records = []

    def run(self, prog, arena, lens, now, off16, stride, prio, now_v=None):
        v = super().run(prog, arena, lens, now, off16, stride, prio, now_v)
        self.records.extend(got_records(*self.dp.li_drain()))
        return v


def run_dual(name, pinned, ora_kind, seed=3):
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    base = scenarios.ALL_SCRIPTS[name]()
    owners = script_owners(base)
    table = make_table(owners)
    script = inject(base, table, seed)
    targets = {o: 100 + j for j, o in enumerate(owners[::3] + [NO_DIR])}
    want = harness.run_script(harness.OracleBackend(ora_kind), script)
    be = DualBackend(table, targets, pinned)
    try:
        got = harness.run_script(be, script)
        harness.compare(want, got, f"{name}: {ora_kind} oracle vs gpu with subscriber_ipv6 filled")
        runs, final = attributions(script, want, ora_kind, table)
    except BaseException:
        be.close()
        raise
    return be, runs, final, targets


# ---------------------------------------------------------------------------
# 1. the golden scripts with IPv6 frames, on every feed
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("script", SCRIPTS)
def test_golden_scripts_dualstack(script, pinned, ora_kind):
    be, runs, final, targets = run_dual(script, pinned, ora_kind)
    try:
        what = f"{script} ({FEED_IDS[FEEDS.index(pinned)]})"
        acct, idle = expected_acct_idle(runs, final)
        check_acct_idle(be.dp, acct, idle, what)
        assert_records_equal(be.records, expected_li(runs, targets), what)
    finally:
        be.close()


def test_zero_copy_chunk_edges(ora_kind):
    """Batches across the zero-copy chunk size, half IPv6, with per-frame clocks."""
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    base = scenarios.ALL_SCRIPTS["pipeline"]()
    owners = script_owners(base)
    table = make_table(owners)
    r = np.random.default_rng(9)
    sc = harness.Script("chunks")
    for st in base.steps:
        if st[0] in ("update", "delete"):
            sc.steps.append(st)
    runs = [st for st in base.steps if st[0] == "run" and st[5] is None and st[1] in PIPES]
    _, prog, arena, lens, now, off16, stride, _, _ = runs[0]
    arena = np.asarray(arena, np.uint8).reshape(-1)
    n0 = len(lens)
    for n in ((1 << 18) - 1, (1 << 18) + 33):
        idx = r.integers(0, n0, n)
        a = arena.reshape(n0, stride)[idx]
        f, l6 = v6_frames(a[:, :12], table, r, n, stride)
        six = r.random(n) < 0.5
        a[six] = f[six]
        l = np.where(six, l6, lens[idx]).astype(np.uint32)
        nv = np.sort(r.integers(now, now + 10**9, n)).astype(np.uint64)
        sc.run(prog, a.reshape(-1), l, now, stride=stride, now_v=nv)
        now += 2 * 10**9
    targets = {owners[0]: 7, owners[1]: 8}
    want = harness.run_script(harness.OracleBackend(ora_kind), sc)
    be = DualBackend(table, targets, True, max_batch=1 << 19, event_capacity=1 << 20)
    try:
        got = harness.run_script(be, sc)
        harness.compare(want, got, "chunk edges")
        rr, final = attributions(sc, want, ora_kind, table)
        assert sum(int(x[3].sum()) for x in rr if x[3] is not None) > 1000, "too few IPv6 frames were attributed"
        acct, idle = expected_acct_idle(rr, final)
        check_acct_idle(be.dp, acct, idle, "chunk edges")
        assert_records_equal(be.records, expected_li(rr, targets), "chunk edges")
    finally:
        be.close()


# ---------------------------------------------------------------------------
# 2. an empty table changes nothing: records, launches and kernel names
# ---------------------------------------------------------------------------
def test_empty_table_is_the_old_behaviour(ora_kind):
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    base = scenarios.ALL_SCRIPTS["pipeline"]()
    table = make_table(script_owners(base))
    script = inject(base, table)
    targets = {o: 1 for o in script_owners(base)[:4]}
    out = []
    for filled in (False, True):
        be = DualBackend([], targets, False)
        try:
            if filled:  # filled, then emptied two ways: delete every entry, and clear
                install(be.dp, table)
                for pl, p, _ in table[: len(table) // 2]:
                    k = np.zeros(1, L.bng_ipv6_prefix_key)
                    k["prefixlen"], k["addr"] = pl, p
                    assert be.dp.delete("subscriber_ipv6", k) == 0
                assert be.dp.clear("subscriber_ipv6") == 0
                assert be.dp.map_info("subscriber_ipv6")["count"] == 0
            be.dp.prof_enable(True)
            n0 = be.dp.launch_count
            got = harness.run_script(be, script)
            out.append((be.dp.launch_count - n0, set(be.dp.prof_read()), be.dp.acct_dump(), be.records, got))
        finally:
            be.close()
    (l0, k0, a0, r0, g0), (l1, k1, a1, r1, g1) = out
    assert l0 == l1 and k0 == k1 and not any("v6" in k for k in k0)
    assert np.array_equal(a0[0], a1[0]) and np.array_equal(a0[1], a1[1])
    assert len(r0) == len(r1) and all(x[0] == y[0] and np.array_equal(x[1], y[1]) for x, y in zip(r0, r1))
    harness.compare(g0, g1, "empty vs emptied table")


def test_ipv6_kernels_only_while_filled():
    with Dataplane(max_subscribers=1 << 10, max_batch=1 << 10) as dp:
        dp.acct_enable("qos_ingress_prog")
        f = np.zeros((4, 64), np.uint8)
        f[:, 12:14] = (0x86, 0xDD)
        lens = np.full(4, 64, np.uint32)
        dp.prof_enable(True)
        dp.run("qos_ingress_prog", f.reshape(-1), lens.copy(), 1, stride=64)
        assert "k_acct" in dp.prof_read() and "k_acct<v6>" not in dp.prof_read()
        install(dp, [(64, _net(1), 0x0100000A)])
        dp.run("qos_ingress_prog", f.reshape(-1), lens.copy(), 2, stride=64)
        assert "k_acct<v6>" in dp.prof_read()


# ---------------------------------------------------------------------------
# 3. the table
# ---------------------------------------------------------------------------
def _key(pl, addr):
    k = np.zeros(1, L.bng_ipv6_prefix_key)
    k["prefixlen"], k["addr"] = pl, addr
    return k


def _val(o):
    return np.array([o], "<u4")


def _lookup(dp, addr, maxlen=128):
    v = dp.lookup("subscriber_ipv6", _key(maxlen, addr))
    return None if v is None else int(v.view("<u4")[0])


def test_table_lifecycle():
    with Dataplane(max_subscribers=64, max_batch=1 << 10) as dp:
        inf = dp.map_info("subscriber_ipv6")
        assert (inf["type"], inf["key_size"], inf["value_size"], inf["max_entries"]) == (11, 20, 4, 128)
        model = []
        r = np.random.default_rng(1)
        probes = sample_addrs(make_table([1, 2, 3]), r, 64)

        def agree(what):
            assert dump_model(dp) == model_of(model), what
            want = np.bincount([m[0] for m in model], minlength=129).astype(np.uint32)
            assert np.array_equal(dp.ipv6_prefix_lengths(), want), f"{what}: per-length counts"
            for a in probes:
                assert _lookup(dp, a) == lpm(model, a), what
                assert _lookup(dp, a, 56) == lpm(model, a, 56), what

        # masked keys: bits past prefixlen are dropped; two spellings of one prefix are one entry
        noisy = _net(3).copy()
        noisy[7:] = 0xAB
        assert dp.update("subscriber_ipv6", _key(48, noisy), _val(3)) == 0
        assert dp.update("subscriber_ipv6", _key(48, _net(3)), _val(4)) == 0
        model.append((48, _net(3), 4))
        agree("masked")
        for bad in (129, 200, 0xFFFFFFFF):
            assert dp.update("subscriber_ipv6", _key(bad, _net(3)), _val(1)) == -errno.EINVAL
            assert dp.delete("subscriber_ipv6", _key(bad, _net(3))) == -errno.EINVAL
            assert dp.update_staged("subscriber_ipv6", _key(bad, _net(3)), _val(1)) == -errno.EINVAL
            with pytest.raises(BngError):
                dp.lookup("subscriber_ipv6", _key(bad, _net(3)))
        # staged and batch updates, nested prefixes, /0 and /128
        t = make_table([11, 12, 13, 14], seed=2)
        for pl, p, o in t[:5]:
            assert dp.update_staged("subscriber_ipv6", _key(pl, p), _val(o)) == 0
        assert dp.update_batch("subscriber_ipv6", np.concatenate([_key(pl, p) for pl, p, _ in t[5:]]),
                               np.concatenate([_val(o) for _, _, o in t[5:]])) == 0
        model += t
        assert dp.update("subscriber_ipv6", _key(0, np.zeros(16, np.uint8)), _val(99)) == 0
        model.append((0, np.zeros(16, np.uint8), 99))
        agree("filled")
        # delete matches (prefixlen, prefix) exactly
        assert dp.delete("subscriber_ipv6", _key(47, _net(3))) == -errno.ENOENT
        assert dp.delete("subscriber_ipv6", _key(48, noisy)) == 0
        model = [m for m in model if not (m[0] == 48 and np.array_equal(m[1], _net(3)))]
        assert dp.delete("subscriber_ipv6", _key(0, np.zeros(16, np.uint8))) == 0
        model = [m for m in model if m[0] != 0]
        agree("deleted")
        # -E2BIG at max_entries
        n = dp.map_info("subscriber_ipv6")["count"]
        fill = [(128, _net(i, hi=0x30), 5) for i in range(128 - n)]
        assert dp.update_batch("subscriber_ipv6", np.concatenate([_key(pl, p) for pl, p, _ in fill]),
                               np.concatenate([_val(o) for *_, o in fill])) == 0
        model += fill
        assert dp.update("subscriber_ipv6", _key(128, _net(999, hi=0x31)), _val(5)) == -errno.E2BIG
        agree("full")
        assert dp.clear("subscriber_ipv6") == 0
        model = []
        agree("cleared")
        assert dp.update("subscriber_ipv6", _key(64, _net(8)), _val(8)) == 0
        model.append((64, _net(8), 8))
        agree("after clear")


# ---------------------------------------------------------------------------
# 4. snapshot / restore, delta replication and failover, hand-over
# ---------------------------------------------------------------------------
def _frames6(addrs, up=True, n_each=3):
    f = np.zeros((len(addrs) * n_each, 64), np.uint8)
    f[:, 12:14] = (0x86, 0xDD)
    f[:, 14] = 0x60
    for j, a in enumerate(addrs):
        f[j * n_each:(j + 1) * n_each, 22 if up else 38:(38 if up else 54)] = a
    return f.reshape(-1), np.full(len(f), 100, np.uint32)


def _subscriber_maps(dp, owners):
    tb = np.zeros(len(owners), L.token_bucket)
    dp.update_batch("qos_ingress", np.array(owners, "<u4").view(np.uint8).reshape(-1, 4), tb)


def _traffic(dp, table, now):
    addrs = [p for _, p, _ in table]
    a, l = _frames6(addrs)
    dp.run("qos_ingress_prog", a, l, now, stride=64)
    a, l = _frames6(addrs, up=False)
    dp.run("qos_egress_prog", a, l, now, stride=64)


def _state(dp):
    k, v = dp.dump("subscriber_ipv6")
    return k.tobytes(), v.tobytes()


def test_snapshot_delta_failover():
    owners = [0x0A000001 + (j << 24) for j in range(6)]
    table = make_table(owners)
    opts = dict(max_subscribers=1 << 10, max_batch=1 << 12)
    with Dataplane(**opts) as a, Dataplane(**opts) as b, Dataplane(**opts) as c:
        for dp in (a, b, c):
            dp.acct_enable("qos_ingress_prog")
            dp.acct_enable("qos_egress_prog")
        _subscriber_maps(a, owners)
        a.delta_enable(True)
        install(a, table[:8])
        b.delta_apply(a.delta_export())
        install(a, table[8:])
        k = _key(table[0][0], table[0][1])
        assert a.delete("subscriber_ipv6", k) == 0
        b.delta_apply(a.delta_export())
        assert _state(b) == _state(a)
        c.restore(a.snapshot())
        assert _state(c) == _state(a)
        for dp in (b, c):
            assert np.array_equal(dp.ipv6_prefix_lengths(), a.ipv6_prefix_lengths())
        # the standby and the restored context attribute as the active does
        for dp in (a, b, c):
            _traffic(dp, table, 10**9)
        assert np.array_equal(a.acct_dump()[1], b.acct_dump()[1]) and np.array_equal(a.acct_dump()[1], c.acct_dump()[1])
        assert int(a.acct_dump()[1]["up_packets"].sum()) > 0
        for pl, p, o in table:
            assert _lookup(b, p) == lpm(table[1:], p)


def test_hand_over():
    owners = [0x0A000001 + (j << 24) for j in range(8)]
    table = make_table(owners)
    opts = dict(max_subscribers=1 << 10, max_batch=1 << 12)
    with Dataplane(**opts) as src, Dataplane(**opts) as dst:
        _subscriber_maps(src, owners)
        install(src, table)
        before = _state(src)
        moved = owners[:3]
        mv = lambda t: [e for e in t if e[2] in moved]  # noqa: E731
        keep = [e for e in table if e[2] not in moved]
        # without detach: nothing changes at the source
        blob = src.sub_export(np.array(moved, "<u4"))
        assert _state(src) == before
        # the blob's subscriber_ipv6 section holds exactly the moved subscribers' prefixes
        assert blob.count(b"subscriber_ipv6") == 1
        # detach removes exactly those
        blob = src.sub_export(np.array(moved, "<u4"), detach=True)
        assert dump_model(src) == model_of(keep)
        assert np.array_equal(src.ipv6_prefix_lengths(), np.bincount([e[0] for e in keep], minlength=129))
        for pl, p, o in table:
            assert _lookup(src, p) == lpm(keep, p)
        assert dst.sub_import(blob) == 0
        assert dump_model(dst) == model_of(mv(table))
        assert np.array_equal(dst.ipv6_prefix_lengths(), np.bincount([e[0] for e in mv(table)], minlength=129))
        for pl, p, o in mv(table):
            assert _lookup(dst, p) == lpm(mv(table), p)
        # the rollback: the blob back into its source restores it exactly
        assert src.sub_import(blob) == 0
        assert _state(src) == before
        # a context without prefixes writes no such section
        with Dataplane(**opts) as plain:
            _subscriber_maps(plain, owners)
            assert b"subscriber_ipv6" not in plain.sub_export(np.array(moved, "<u4"))
