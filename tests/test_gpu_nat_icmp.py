"""ICMP error translation in nat44_ingress (bng_nat_icmp_errors_enable, include/bng_b200.h): an inbound Destination
Unreachable, Time Exceeded or Parameter Problem is DNATed to the subscriber whose flow it quotes.

The oracle has no such rule, so the expected results combine two runs.  The rule reads only the existence of a reverse
entry and its session and the session's immutable orig_ip / orig_port, and changes no table, counter or record; the
only table change nat44_ingress makes is erasing stale reverse entries, whose error frames pass either way.  So:
  - the oracle's nat44_ingress runs on the batch with the ICMP error frames removed, and
  - the rule, restated below in numpy, runs on the error frames against the oracle's table dumps taken at the start
    of the batch, giving each error frame's bytes and its packets_dnat / packets_passed count.
The flows are made by the oracle's nat44_egress, and the errors quote the oracle's own SNATed frames.  A CPU test
checks the restatement against two properties that do not depend on it: a translated error quotes the subscriber's
original frame, and its checksums stay valid."""
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
from bng_b200 import synth as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FEEDS = [False, True, "device"]
FEED_IDS = ["pageable", "pinned", "device"]
ERR_TYPES = (3, 11, 12)
STRIDE = 128
ROUTER = 0xC0000201  # 192.0.2.1: a third-party router on the path
N_SUBS = 12
T0 = 5_000_000_000


def _need(kind):
    if kind == "none":
        pytest.fail("no oracle library present on this box")


# ---------------------------------------------------------------------------
# the rule, restated
# ---------------------------------------------------------------------------
def rd16(f, o):
    return int(f[o]) | (int(f[o + 1]) << 8)


def rd32(f, o):
    return rd16(f, o) | (rd16(f, o + 2) << 16)


def wr16(f, o, v):
    f[o], f[o + 1] = v & 0xFF, (v >> 8) & 0xFF


def _fold(c):
    c = (c & 0xFFFF) + (c >> 16)
    c = (c & 0xFFFF) + (c >> 16)
    return ~c & 0xFFFF


def upd32(ck, old, new):
    return _fold((~ck & 0xFFFF) + (~old & 0xFFFF) + (~(old >> 16) & 0xFFFF) + (new & 0xFFFF) + (new >> 16))


def upd16(ck, old, new):
    return _fold((~ck & 0xFFFF) + (~old & 0xFFFF) + (new & 0xFFFF))


def flow_tables(dump_rev, dump_ses):
    """{reverse key[:13]: session key[:13]} and {session key[:13]: (orig_ip bytes, orig_port bytes)}."""
    rev = {bytes(k[:13]): bytes(v[:13]) for k, v in zip(*dump_rev)}
    ses = {bytes(k[:13]): (bytes(v[8:12]), bytes(v[6:8])) for k, v in zip(*dump_ses)}
    return rev, ses


def is_error_frame(f, present):
    """An ICMP error frame: untagged IPv4, protocol 1, type 3 / 11 / 12, the 8-byte ICMP header present."""
    if present < 34 or f[12] != 0x08 or f[13] != 0x00 or f[23] != 1:
        return False
    l4 = 14 + (f[14] & 0x0F) * 4
    return l4 + 8 <= present and int(f[l4]) in ERR_TYPES


def translate(f, present, rev, ses):
    """The rule on one ICMP error frame f (u8 array, changed in place): True when translated."""
    ip = int(f[51])
    if f[14] != 0x45 or f[42] != 0x45 or ip not in (6, 17, 1) or bytes(f[54:58]) != bytes(f[30:34]):
        return False
    if present < (68 if ip == 1 else 66):
        return False
    pp = (66 if ip == 1 else 62)
    key = bytes(f[58:62]) + bytes(f[54:58]) + (b"\0\0" if ip == 1 else bytes(f[64:66])) + bytes(f[pp:pp + 2]) + bytes([ip])
    ok = rev.get(key)
    if ok is None or ok not in ses:
        return False
    oip_b, oport_b = ses[ok]
    isrc, oip = rd32(f, 54), int.from_bytes(oip_b, "little")
    pport, oport = rd16(f, pp), int.from_bytes(oport_b, "little")
    f[30:34] = np.frombuffer(oip_b, np.uint8)
    wr16(f, 24, upd32(rd16(f, 24), isrc, oip))
    ihc = rd16(f, 52)
    ihc2 = upd32(ihc, isrc, oip)
    f[54:58] = np.frombuffer(oip_b, np.uint8)
    wr16(f, 52, ihc2)
    ic = upd32(rd16(f, 36), isrc, oip)
    ic = upd16(ic, ihc, ihc2)
    ic = upd16(ic, pport, oport)
    wr16(f, pp, oport)
    at = 64 if ip == 1 else (68 if ip == 17 and present >= 70 and rd16(f, 68) else (78 if ip == 6 and present >= 80 else 0))
    if at:
        k0 = rd16(f, at)
        k1 = upd16(k0, pport, oport) if ip == 1 else upd16(upd32(k0, isrc, oip), pport, oport)
        if ip == 17 and k1 == 0:
            k1 = 0xFFFF
        wr16(f, at, k1)
        ic = upd16(ic, k0, k1)
    wr16(f, 36, ic)
    return True


def layout(lens, off16, stride):
    n = len(lens)
    starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(n, dtype=np.int64) * stride
    present = lens.astype(np.int64) if off16 is not None else np.minimum(lens.astype(np.int64), stride)
    return starts, present


class RuleOracle(harness.OracleBackend):
    """The oracle, with nat44_ingress run as described at the top while `on`."""

    def __init__(self, kind, on=True):
        super().__init__(kind)
        self.on = on
        self.dnat = self.passed = 0  # the error frames' counts
        self.translated = []  # per nat44_ingress run: indices of the translated frames

    def run(self, prog, arena, lens, now, off16, stride, prio, now_v=None):
        if prog != "nat44_ingress" or not self.on:
            return super().run(prog, arena, lens, now, off16, stride, prio, now_v)
        starts, present = layout(lens, off16, stride)
        rev, ses = flow_tables(self.o.dump("nat_reverse"), self.o.dump("nat_sessions"))
        err = np.array([is_error_frame(arena[s:s + 100], p) for s, p in zip(starts, present)], bool)
        done = []
        for i in np.nonzero(err)[0]:
            s = int(starts[i])
            f = arena[s:s + 96].copy()
            if translate(f, int(present[i]), rev, ses):
                arena[s:s + 96] = f
                done.append(int(i))
        self.dnat += len(done)
        self.passed += int(err.sum()) - len(done)
        self.translated.append(np.array(done, np.int64))
        keep = np.nonzero(~err)[0]
        verdict = np.full(len(lens), L.TC_ACT_OK, np.uint8)
        if len(keep):
            assert not (starts % 16).any() and (present[keep] == lens[keep]).all(), "the oracle runs kept frames by len"
            oa = self.o.arena(len(arena) + 64)
            oa[:len(arena)] = arena
            oa[len(arena):] = 0
            l = lens[keep].copy()
            nv = None if now_v is None else np.ascontiguousarray(now_v[keep])
            verdict[keep] = self.o.run(prog, oa, l, now, off16=(starts[keep] // 16).astype(np.uint32), now_v=nv)
            arena[:] = oa[:len(arena)]
            self.o.free_arenas()
        return verdict

    def stats(self, m):
        s = super().stats(m)
        if m == "nat_stats_map":
            s = s.copy()
            s[list(L.nat_stats.names).index("packets_dnat")] += self.dnat
            s[list(L.nat_stats.names).index("packets_passed")] += self.passed
        return s


# ---------------------------------------------------------------------------
# flows and frames
# ---------------------------------------------------------------------------
def flows(r, n_subs=N_SUBS, per=6):
    """The subscribers' original (pre-SNAT) frames, u8[n, 64]: TCP, UDP with and without a checksum, ICMP echo."""
    sub = np.repeat(np.arange(n_subs), per)
    n = len(sub)
    kind = np.tile(np.arange(per), n_subs) % 4
    proto = np.array([6, 17, 17, 1], np.uint32)[kind]
    sport = (20000 + np.arange(n)).astype(np.uint32)
    dport = np.array([443, 53, 123, 0], np.uint32)[kind]
    dst = (np.uint32(0x08080000) + r.integers(0, 4, n).astype(np.uint32)).astype(np.uint32)
    ck = r.integers(1, 65536, n).astype(np.uint32)
    ck[kind == 2] = 0  # UDP without a checksum
    hdr = S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), dst, proto, sport, dport,
                         np.full(n, 64, np.uint32), l4_check=ck, tcp_flags=0x02)
    return hdr


def inet_csum(b):
    b = np.asarray(b, np.uint32)
    if len(b) % 2:
        b = np.append(b, 0)
    s = int((b[0::2] << 8 | b[1::2]).sum())
    while s >> 16:
        s = (s & 0xFFFF) + (s >> 16)
    return s  # 0xFFFF: valid


def error_frame(snat, qlen, typ, code, mtu=0):
    """An ICMP error from ROUTER to the quoted packet's source, quoting the first qlen bytes of the IPv4 packet in
    snat (a frame as nat44_egress left it).  Valid checksums.  Returns (u8[STRIDE], len)."""
    f = np.zeros(STRIDE, np.uint8)
    f[0:6], f[6:12] = snat[6:12], snat[0:6]
    f[12:14] = (0x08, 0x00)
    f[14] = 0x45
    f[16:18] = S.port_bytes(20 + 8 + qlen)
    f[22], f[23] = 64, 1
    f[26:30] = S.ip_bytes(ROUTER)
    f[30:34] = snat[26:30]
    f[24:26] = S.ip_checksum(f[None, 14:34])[0]
    f[34], f[35] = typ, code
    if mtu:
        f[40:42] = S.port_bytes(mtu)
    if typ == 12:
        f[38] = 9  # pointer
    f[42:42 + qlen] = snat[14:14 + qlen]
    c = ~inet_csum(f[34:42 + qlen]) & 0xFFFF
    f[36:38] = (c >> 8, c & 0xFF)
    return f, 42 + qlen


def random_error(r, snat):
    typ = int(r.choice(ERR_TYPES))
    code = int(r.integers(0, 16)) if typ == 3 else int(r.integers(0, 2))
    return error_frame(snat, int(r.choice([28, 48, 50])), typ, code, 1492 if (typ == 3 and code == 4) else 0)


def replies(snat, r):
    """Ordinary replies to the SNATed frames, with TCP SYN-ACK / ACK / FIN / RST."""
    out = np.zeros((len(snat), STRIDE), np.uint8)
    out[:, :64] = snat
    out[:, 26:30], out[:, 30:34] = snat[:, 30:34], snat[:, 26:30]
    tu = (snat[:, 23] == 6) | (snat[:, 23] == 17)
    out[tu, 34:36], out[tu, 36:38] = snat[tu, 36:38], snat[tu, 34:36]
    icmp = snat[:, 23] == 1
    out[icmp, 34] = 0  # echo reply
    tcp = snat[:, 23] == 6
    out[tcp, 47] = r.choice(np.array([0x12, 0x10, 0x11, 0x04], np.uint8), int(tcp.sum()))
    return out, np.full(len(snat), 64, np.uint32)


def not_translatable(r, snat, pubs):
    """Error frames the rule must pass unchanged, one kind per row of the list."""
    out = []
    for j in range(len(snat)):
        f, l = random_error(r, snat[j])
        k = j % 9
        if k == 0:  # reverse miss: another destination port (or ICMP id) in the quote
            f[66 if f[51] == 1 else 64] ^= 0x5A
        elif k == 1:  # outer destination is not the quoted source
            f[30:34] = S.ip_bytes(pubs[-1] + 7)
        elif k == 2:  # options in the outer header: the ICMP message moves 4 bytes on
            g = np.zeros(STRIDE, np.uint8)
            g[:34], g[34:38], g[38:STRIDE] = f[:34], 1, f[34:STRIDE - 4]
            g[14] = 0x46
            f, l = g, l + 4
        elif k == 3:  # options in the quoted header
            f[42] = 0x46
        elif k == 4:  # quoted version 6
            f[42] = 0x65
        elif k == 5:  # quoted protocol 47
            f[51] = 47
        elif k == 6:  # deprecated source quench / redirect: not error frames, today's path
            f[34] = 4 if j % 2 else 5
        elif k == 7:  # the quoted header cut short
            l = 42 + int(r.integers(8, 24))
        else:  # reverse miss: another public port (or ICMP id) in the quote
            f[67 if f[51] == 1 else 63] ^= 0x33
        out.append((f, l))
    return out


def base_script(seed=0x1C3E, n_subs=N_SUBS, per=6, stale_every=5):
    """Maps, one nat44_egress batch of every subscriber's flows, then the sessions of every stale_every-th TCP flow
    deleted underneath nat_reverse.  Returns (script, original frames, public addresses, egress step tag)."""
    r = np.random.default_rng(seed)
    sc = harness.Script("nat_icmp")
    pubs = scenarios.nat_maps(sc, n_subs, 64, 0x0F)
    orig = flows(r, n_subs, per)
    sc.run("nat44_egress", scenarios.fixed(orig), np.full(len(orig), 64, np.uint32), T0)
    tag = f"s{len(sc.steps) - 1:03d}"
    tcp = np.nonzero(orig[:, 23] == 6)[0][::stale_every]
    k = np.zeros(len(tcp), L.nat_key)
    k["src_ip"], k["dst_ip"] = orig[tcp, 26:30], orig[tcp, 30:34]
    k["src_port"], k["dst_port"], k["protocol"] = orig[tcp, 34:36], orig[tcp, 36:38], 6
    for x in k:
        sc.delete("nat_sessions", x)
    return sc, orig, pubs, tag


def snat_of(res, tag):
    return res[tag + "_frames"].reshape(-1, 64)


def mixed(res, tag, seed, pubs, now, frame_clock=False, errors=True, bad=True, stride=STRIDE, copies=4):
    """A batch of ordinary replies to every flow interleaved with errors quoting the same flows (and the stale ones),
    plus the untranslatable kinds; shuffled."""
    r = np.random.default_rng(seed)
    snat = snat_of(res, tag)
    rows, lens = [], []
    for _ in range(copies):
        f, l = replies(snat, r)
        rows += list(f)
        lens += list(l)
        if errors:
            for s in snat:
                f, l = random_error(r, s)
                rows.append(f)
                lens.append(l)
    if bad:
        for f, l in not_translatable(r, snat, pubs):
            rows.append(f)
            lens.append(l)
    order = r.permutation(len(rows))
    a = np.stack(rows)[order][:, :stride]
    lens = np.array(lens, np.uint32)[order]
    d = {"arena": a.reshape(-1).copy(), "lens": lens, "now_ns": now, "stride": stride}
    if frame_clock:
        d["now_v"] = (now + np.sort(r.integers(0, 500_000, len(lens)))).astype(np.uint64)
    return d


def script_with(kind, frame_clock=False, **kw):
    sc, orig, pubs, tag = base_script(**kw)
    sc.run_from("nat44_ingress", lambda res: mixed(res, tag, 1, pubs, T0 + 10**9, frame_clock))
    sc.run_from("nat44_ingress", lambda res: mixed(res, tag, 2, pubs, T0 + 2 * 10**9, frame_clock))
    return sc, orig, pubs, tag


class IcmpBackend(harness.GpuBackend):
    def __init__(self, pinned=False, on=True, **opts):
        super().__init__(pinned=pinned, **opts)
        if on:
            self.dp.nat_icmp_errors_enable(True)


def check(sc, kind, pinned, what, **opts):
    ora = RuleOracle(kind)
    want = harness.run_script(ora, sc)
    be = IcmpBackend(pinned, **opts)
    try:
        got = harness.run_script(be, sc)
    finally:
        be.close()
    harness.compare(want, got, f"{what}: {kind} oracle with the rule restated vs gpu")
    return want, ora


# ---------------------------------------------------------------------------
# 1. the restatement, checked without a GPU
# ---------------------------------------------------------------------------
def test_restatement_quotes_the_original(ora_kind):
    """Every translated error quotes the subscriber's original frame (IPv4 header and 8 L4 bytes, up to a checksum
    0x0000 / 0xFFFF), is addressed to it, and keeps valid checksums where they were valid and whole."""
    _need(ora_kind)
    sc, orig, pubs, tag = script_with(ora_kind)
    ora = RuleOracle(ora_kind)
    res = harness.run_script(ora, sc)
    runs = [k for k in sorted(res) if k.endswith("_frames")][1:]
    assert ora.dnat > 500 and ora.passed > 50, (ora.dnat, ora.passed)
    snat = snat_of(res, tag)
    for k, done in zip(runs, ora.translated):
        a = res[k].reshape(-1, STRIDE)
        lens = res[k.replace("_frames", "_len")]
        for i in done:
            f = a[i]
            ip = int(f[51])
            want = None
            for jj in range(len(orig)):
                o = orig[jj]
                if o[23] == ip and (o[26:30] == f[54:58]).all() and (o[30:34] == f[58:62]).all() and \
                        ((o[38:40] == f[66:68]).all() if ip == 1 else (o[34:38] == f[62:66]).all()):
                    want = o
                    break
            assert want is not None, f"{k} frame {i}: quotes no original flow"
            q, w = f[42:70].copy(), want[14:42].copy()
            for c in (10, {17: 26, 1: 22}.get(ip)):  # the quoted IPv4 checksum, and the UDP / ICMP checksum
                if c is not None and {rd16(q, c), rd16(w, c)} == {0, 0xFFFF}:
                    q[c:c + 2] = w[c:c + 2]
            assert np.array_equal(q, w), f"{k} frame {i}: quote differs from the original"
            assert (f[30:34] == want[26:30]).all()
            assert inet_csum(f[14:34]) == 0xFFFF and inet_csum(f[42:62]) == 0xFFFF
            assert inet_csum(f[34:int(lens[i])]) == 0xFFFF, f"{k} frame {i}: ICMP checksum"


# ---------------------------------------------------------------------------
# 2. against the GPU
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("clock", ["batch", "frame"])
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
def test_mixed_batches(pinned, clock, ora_kind):
    _need(ora_kind)
    sc, _, _, _ = script_with(ora_kind, frame_clock=clock == "frame")
    want, ora = check(sc, ora_kind, pinned, f"mixed ({FEED_IDS[FEEDS.index(pinned)]}, {clock} clock)")
    assert ora.dnat > 500 and ora.passed > 50
    assert want["st_nat_stats_map"][list(L.nat_stats.names).index("sessions_expired")] > 0  # stale erased by replies


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
def test_lengths_and_rings(pinned, ora_kind):
    """Every length from 34 to 100 bytes on errors quoting live flows, and the same errors through a 64-byte
    header-split ring, which holds no quoted port: those pass unchanged."""
    _need(ora_kind)
    sc, orig, pubs, tag = base_script(stale_every=1000)

    def lengths(res, stride):
        r = np.random.default_rng(3)
        snat = snat_of(res, tag)
        rows, lens = [], []
        for l in range(34, 101):
            for s in snat[r.permutation(len(snat))[:6]]:
                f, _ = random_error(r, s)
                rows.append(f[:stride])
                lens.append(l)
        return {"arena": np.stack(rows).reshape(-1).copy(), "lens": np.array(lens, np.uint32), "now_ns": T0 + 10**9,
                "stride": stride}

    sc.run_from("nat44_ingress", lambda res: lengths(res, STRIDE))
    sc.run_from("nat44_ingress", lambda res: lengths(res, 64))
    want, ora = check(sc, ora_kind, pinned, f"lengths ({FEED_IDS[FEEDS.index(pinned)]})")
    assert len(ora.translated[0]) > 100 and len(ora.translated[1]) == 0


@pytest.mark.gpu
def test_zero_copy_chunk_edges(ora_kind):
    """Errors on both sides of the 2^18-frame chunk edges of the pinned feed."""
    _need(ora_kind)
    sc, orig, pubs, tag = base_script(stale_every=1000)

    def big(res, n, seed):
        r = np.random.default_rng(seed)
        snat = snat_of(res, tag)
        rep, rl = replies(snat, r)
        pick = r.integers(0, len(snat), n)
        a = rep[pick].copy()
        lens = rl[pick].copy()
        edge = np.zeros(n, bool)
        for e in range(1 << 18, n, 1 << 18):
            edge[max(0, e - 40):e + 40] = True
        sel = np.nonzero(edge | (r.random(n) < 0.01))[0]
        for i in sel:
            a[i], lens[i] = random_error(r, snat[pick[i]])
        return {"arena": a.reshape(-1).copy(), "lens": lens, "now_ns": T0 + seed * 10**9, "stride": STRIDE,
                "now_v": (T0 + seed * 10**9 + np.sort(r.integers(0, 10**8, n))).astype(np.uint64)}

    sc.run_from("nat44_ingress", lambda res: big(res, (1 << 18) + 77, 1))
    sc.run_from("nat44_ingress", lambda res: big(res, (1 << 19) + 5, 2))
    _, ora = check(sc, ora_kind, True, "chunk edges", max_batch=1 << 20)
    assert ora.dnat > 5000


# ---------------------------------------------------------------------------
# 3. off is today
# ---------------------------------------------------------------------------
def _observe(sc, setup):
    be = harness.GpuBackend(pinned=False)
    try:
        setup(be.dp)
        be.dp.prof_enable(True)
        n0 = be.dp.launch_count
        got = harness.run_script(be, sc)
        return be.dp.launch_count - n0, set(be.dp.prof_read()), got
    finally:
        be.close()


@pytest.mark.gpu
def test_off_is_today(ora_kind):
    _need(ora_kind)
    sc, _, _, _ = script_with(ora_kind)
    today = harness.run_script(harness.OracleBackend(ora_kind), sc)  # errors keyed by bytes 4-5, as ever
    never = _observe(sc, lambda dp: None)
    harness.compare(today, never[2], "never set: oracle vs gpu")
    assert "k_nat_ingress" in never[1] and not any("icmperr" in k for k in never[1])

    def on_off(dp):
        dp.nat_icmp_errors_enable(True)
        dp.nat_icmp_errors_enable(False)

    again = _observe(sc, on_off)
    harness.compare(today, again[2], "on, then off: oracle vs gpu")
    assert again[:2] == never[:2]
    # with no error frames in the batches, "on" computes what "off" does
    quiet, _, pubs, tag = base_script()
    quiet.run_from("nat44_ingress", lambda res: mixed(res, tag, 5, pubs, T0 + 10**9, errors=False, bad=False))
    on = _observe(quiet, lambda dp: dp.nat_icmp_errors_enable(True))
    harness.compare(harness.run_script(harness.OracleBackend(ora_kind), quiet), on[2], "on, no errors: oracle vs gpu")
    assert "k_nat_ingress<icmperr>" in on[1] and "k_nat_ingress" not in on[1]


# ---------------------------------------------------------------------------
# 4. attribution: accounting, idle stamps and interception see the translated frame
# ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_attribution(ora_kind):
    _need(ora_kind)
    sc, orig, pubs, tag = base_script(stale_every=1000)
    sc.run_from("nat44_ingress", lambda res: mixed(res, tag, 7, pubs, T0 + 10**9, copies=1))
    ora = RuleOracle(ora_kind)
    want = harness.run_script(ora, sc)
    subs = S.ip_bytes(S.sub_ip(np.arange(N_SUBS)))
    sub_words = subs.copy().view("<u4").reshape(-1)
    be = IcmpBackend(False)
    try:
        dp = be.dp
        dp.acct_enable("nat44_ingress")
        dp.idle_enable("nat44_ingress")
        dp.li_configure()
        for j, w in enumerate(sub_words[:4]):
            dp.li_target_set(int(w), 50 + j)
        got = harness.run_script(be, sc)
        harness.compare(want, got, "attribution run")
        acct, found = dp.acct_read(subs)
        idle, _ = dp.idle_read(subs)
        hdr, data = dp.li_drain()
    finally:
        be.close()
    assert found.all()
    k = [x for x in sorted(want) if x.endswith("_frames")][-1]
    a = want[k].reshape(-1, STRIDE)
    lens = want[k.replace("_frames", "_len")]
    dst = a[:, 30:34].copy().view("<u4").reshape(-1)
    done = set(ora.translated[-1].tolist())
    assert len(done) > 50
    for j, w in enumerate(sub_words):
        mine = np.nonzero(dst == w)[0]
        assert acct[j]["down_packets"] == len(mine) and acct[j]["down_bytes"] == int(lens[mine].sum()), j
        assert any(i in done for i in mine), f"subscriber {j} was sent no translated error"
        assert idle[j]["down_ns"] == T0 + 10**9
    # untranslated errors stay addressed to a public address, which is nobody's
    err_passed = [i for i in range(len(a)) if is_error_frame(a[i], min(int(lens[i]), STRIDE)) and i not in done]
    assert err_passed and not np.isin(dst[err_passed], sub_words).any()
    # captured after DNAT: exactly the frames to the targets, as they left the program
    tgt = np.nonzero(np.isin(dst, sub_words[:4]))[0]
    down = hdr["dir"] == 1
    hdr, data = hdr[down], [d for d, x in zip(data, down) if x]
    assert list(hdr["frame"]) == list(tgt)
    for h, d in zip(hdr, data):
        i = int(h["frame"])
        assert np.array_equal(d, a[i, :len(d)]), i
    assert any(int(h["frame"]) in done for h in hdr)


# ---------------------------------------------------------------------------
# 5. the interface (no GPU)
# ---------------------------------------------------------------------------
def test_header_declares_the_call():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bng_b200.h")).read(), flags=re.S)
    assert re.search(r"int\s+bng_nat_icmp_errors_enable\s*\(\s*bng_ctx\s*\*\s*ctx\s*,\s*int\s+on\s*\)\s*;", src)


def test_binding_exposes_the_call():
    assert "bng_nat_icmp_errors_enable" in D.EXPORTED_SYMBOLS
    assert callable(Dataplane.nat_icmp_errors_enable)


def test_null_context_is_einval():
    lib = D.load_library()
    assert lib.bng_nat_icmp_errors_enable(None, 1) == -errno.EINVAL
    assert lib.bng_nat_icmp_errors_enable(None, 0) == -errno.EINVAL
