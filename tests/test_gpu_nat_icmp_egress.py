"""Upstream ICMP error translation in nat44_egress, pipeline_up and pipeline_tc (bng_nat_icmp_errors_egress_enable,
include/bng_b200.h): a subscriber's Destination Unreachable, Time Exceeded or Parameter Problem about a frame it
received leaves from its public address, quoting the public address and port of the flow.

The oracle has no such rule, and the rule depends on the frame's place in the batch (a flow created by an earlier frame
of the same subscriber is seen).  So the expected results are built stage by stage, as tests/test_gpu_qos_v6.py does:
antispoof, then NAT, then the token bucket over the survivors keyed on the pre-NAT source (in pipeline_tc the bucket
runs before NAT).  The NAT stage runs the oracle's nat44_egress in segments split at each error frame the rule looks
at; before each such frame the rule, restated in numpy, reads the oracle's nat_sessions dump at that point.  A
translated error is rewritten by the restatement, left out of the oracle's input and counted in packets_snat; an
untranslated one goes to the oracle as it is.  The flows are made by the oracle's nat44_egress and the replies DNATed
by its nat44_ingress; the errors quote those replies as the subscriber received them.  A CPU test checks the
restatement against properties that do not depend on it."""
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
PROGS = ["nat44_egress", "pipeline_up", "pipeline_tc"]
ERR_TYPES = (3, 11, 12)
STRIDE = 128
N_SUBS = 14  # the last one has no subscriber_nat entry
T0 = 5_000_000_000
NATF_HAIRPIN = 0x04
SNAT = list(L.nat_stats.names).index("packets_snat")
HAIRPIN = list(L.nat_stats.names).index("packets_hairpin")


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


def is_private(f):
    a, b = int(f[26]), int(f[27])
    return a == 10 or (a == 172 and 16 <= b <= 31) or (a == 192 and b == 168) or (a == 100 and 64 <= b <= 127)


def is_error_frame(f, present):
    """The frames the rule looks at: untagged IPv4 without options, protocol 1, type 3 / 11 / 12, ICMP header present."""
    return present >= 42 and f[12] == 0x08 and f[13] == 0x00 and (f[14] & 0x0F) == 5 and f[23] == 1 and \
        int(f[34]) in ERR_TYPES


def sessions(dump):
    """{session key[:13]: (nat_ip bytes, nat_port bytes)}"""
    return {bytes(k[:13]): (bytes(v[0:4]), bytes(v[4:6])) for k, v in zip(*dump)}


def translate(f, present, ses):
    """The rule on one ICMP error frame f (u8 array of at least 80 bytes, changed in place): True when translated."""
    ip = int(f[51])
    if f[42] != 0x45 or ip not in (6, 17, 1) or bytes(f[58:62]) != bytes(f[26:30]):
        return False
    if present < (68 if ip == 1 else 66):
        return False
    pp = 66 if ip == 1 else 64
    key = bytes(f[58:62]) + bytes(f[54:58]) + bytes(f[pp:pp + 2]) + (b"\0\0" if ip == 1 else bytes(f[62:64])) + bytes([ip])
    hit = ses.get(key)
    if hit is None:
        return False
    nip_b, nport_b = hit
    sub, nip = rd32(f, 26), int.from_bytes(nip_b, "little")
    pport, nport = rd16(f, pp), int.from_bytes(nport_b, "little")
    f[26:30] = np.frombuffer(nip_b, np.uint8)
    wr16(f, 24, upd32(rd16(f, 24), sub, nip))
    ihc = rd16(f, 52)
    ihc2 = upd32(ihc, sub, nip)
    f[58:62] = np.frombuffer(nip_b, np.uint8)
    wr16(f, 52, ihc2)
    ic = upd32(rd16(f, 36), sub, nip)
    ic = upd16(ic, ihc, ihc2)
    ic = upd16(ic, pport, nport)
    wr16(f, pp, nport)
    at = 64 if ip == 1 else (68 if ip == 17 and present >= 70 and rd16(f, 68) else (78 if ip == 6 and present >= 80 else 0))
    if at:
        k0 = rd16(f, at)
        k1 = upd16(k0, pport, nport) if ip == 1 else upd16(upd32(k0, sub, nip), pport, nport)
        if ip == 17 and k1 == 0:
            k1 = 0xFFFF
        wr16(f, at, k1)
        ic = upd16(ic, k0, k1)
    wr16(f, 36, ic)
    return True


class RuleOracle(harness.OracleBackend):
    """The oracle with nat44_egress, pipeline_up and pipeline_tc run as described at the top while `on`."""

    def __init__(self, kind, on=True):
        super().__init__(kind)
        self.on = on
        self.snat = self.hairpin = 0
        self.translated = []  # per run of a program with a NAT stage: indices of the translated frames

    def run(self, prog, arena, lens, now, off16, stride, prio, now_v=None):
        if prog not in PROGS or not self.on or (off16 is None and stride < 66):
            # (a ring of slots shorter than 66 bytes holds no translatable error: the oracle as it is)
            if prog in PROGS and self.on:
                self.translated.append(np.zeros(0, np.int64))
            return super().run(prog, arena, lens, now, off16, stride, prio, now_v)
        n = len(lens)
        starts = off16.astype(np.int64) * 16 if off16 is not None else np.arange(n, dtype=np.int64) * stride
        assert not (starts % 16).any(), "the stages address frames by 16-byte offsets"
        present = lens.astype(np.int64) if off16 is not None else np.minimum(lens.astype(np.int64), stride)
        oa = self.o.arena(len(arena) + 128)
        oa[:len(arena)] = arena
        oa[len(arena):] = 0
        subs = {bytes(k) for k in self.o.dump("subscriber_nat")[0]}
        hp = {bytes(k) for k in self.o.dump("hairpin_ips")[0]}
        flags = int(self.o.lookup("nat_config_map", np.zeros(4, np.uint8))[:4].view("<u4")[0])
        done = []

        def stage(p, idx, data):
            if len(idx) == 0:
                return np.zeros(0, np.uint8)
            assert (present[idx] == lens[idx]).all(), "the oracle runs subsets by len"
            l = lens[idx].copy()
            pr = None if prio is None else prio[idx].copy()
            nv = None if now_v is None else np.ascontiguousarray(now_v[idx])
            v = self.o.run(p, data, l, now, off16=(starts[idx] // 16).astype(np.uint32), priority=pr, now_v=nv)
            lens[idx] = l
            if pr is not None:
                prio[idx] = pr
            return v

        def nat(idx):
            v = np.full(len(idx), L.TC_ACT_OK, np.uint8)
            pend, ses = [], None
            for j, i in enumerate(idx):
                s = int(starts[i])
                f = oa[s:s + 100]
                if is_error_frame(f, present[i]) and is_private(f) and bytes(f[26:30]) in subs:
                    if pend:
                        v[pend] = stage("nat44_egress", idx[pend], oa)
                        pend, ses = [], None
                    if ses is None:
                        ses = sessions(self.o.dump("nat_sessions"))
                    g = oa[s:s + 96].copy()
                    if translate(g, int(present[i]), ses):
                        oa[s:s + 96] = g
                        done.append(int(i))
                        self.snat += 1
                        self.hairpin += bool(flags & NATF_HAIRPIN) and bytes(f[30:34]) in hp
                        continue
                pend.append(j)
            if pend:
                v[pend] = stage("nat44_egress", idx[pend], oa)
            return v

        verdict = np.zeros(n, np.uint8)
        everyone = np.arange(n)
        shot = L.TC_ACT_SHOT
        if prog == "nat44_egress":
            verdict[:] = nat(everyone)
        else:
            v = stage("antispoof_ingress", everyone, oa)
            verdict[v == shot] = shot
            s1 = everyone[v != shot]
            if prog == "pipeline_up":
                pre = self.o.arena(len(oa))
                pre[:] = oa  # qos_ingress_prog keys on the frame as it entered NAT
                v = nat(s1)
                verdict[s1[v == shot]] = shot
                s2 = s1[v != shot]
                v = stage("qos_ingress_prog", s2, pre)
                verdict[s2[v == shot]] = shot
            else:
                v = stage("qos_ingress_prog", s1, oa)
                verdict[s1[v == shot]] = shot
                s2 = s1[v != shot]
                v = nat(s2)
                verdict[s2[v == shot]] = shot
        arena[:] = oa[:len(arena)]
        self.o.free_arenas()
        self.translated.append(np.array(sorted(done), np.int64))
        return verdict

    def stats(self, m):
        s = super().stats(m)
        if m == "nat_stats_map":
            s = s.copy()
            s[SNAT] += self.snat
            s[HAIRPIN] += self.hairpin
        return s


# ---------------------------------------------------------------------------
# flows and frames
# ---------------------------------------------------------------------------
def inet_csum(b):
    b = np.asarray(b, np.uint32)
    if len(b) % 2:
        b = np.append(b, 0)
    s = int((b[0::2] << 8 | b[1::2]).sum())
    while s >> 16:
        s = (s & 0xFFFF) + (s >> 16)
    return s  # 0xFFFF: valid


def flows(r, n_subs=N_SUBS, per=6, sport0=20000):
    """The subscribers' original frames, u8[n, 64] (valid IPv4 and L4 checksums): TCP, UDP with and without a
    checksum, ICMP echo."""
    sub = np.repeat(np.arange(n_subs), per)
    n = len(sub)
    kind = np.tile(np.arange(per), n_subs) % 4
    proto = np.array([6, 17, 17, 1], np.uint32)[kind]
    sport = (sport0 + np.arange(n)).astype(np.uint32)
    dport = np.array([443, 53, 123, 0], np.uint32)[kind]
    dst = (np.uint32(0x08080000) + r.integers(0, 4, n).astype(np.uint32)).astype(np.uint32)
    hdr = S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), dst, proto, sport, dport,
                         np.full(n, 64, np.uint32), l4_check=np.zeros(n, np.uint32), tcp_flags=0x02)
    for i in range(n):
        f = hdr[i]
        f[24:26] = 0
        f[24:26] = S.ip_checksum(f[None, 14:34])[0]
        at = {6: 50, 17: 40, 1: 36}[int(f[23])]
        if kind[i] == 2:
            continue  # UDP without a checksum
        f[at:at + 2] = 0
        body = f[34:64]
        if f[23] == 1:
            c = ~inet_csum(body) & 0xFFFF
        else:
            ph = np.concatenate([f[26:34], [0, f[23]], S.port_bytes(30)]).astype(np.uint8)
            c = ~inet_csum(np.concatenate([ph, body])) & 0xFFFF
            if f[23] == 17 and c == 0:
                c = 0xFFFF
        f[at:at + 2] = (c >> 8, c & 0xFF)
    return hdr


def reply_of(f):
    """The remote's reply to a subscriber's frame f, as the subscriber receives it (before or without NAT): the
    addresses and ports swapped, an ICMP echo reply for an echo request."""
    g = f.copy()
    g[0:6], g[6:12] = f[6:12], f[0:6]
    g[26:30], g[30:34] = f[30:34], f[26:30]
    if f[23] == 1:
        g[34] = 0
        wr16(g, 36, upd16(rd16(g, 36), 0x0008, 0x0000))
    else:
        g[34:36], g[36:38] = f[36:38], f[34:36]
    return g


def sub_error(rcv, qlen, typ, code, mtu=0):
    """The subscriber's ICMP error about the frame rcv it received (as delivered to it), quoting rcv's IPv4 header and
    the first qlen - 20 bytes after it.  Valid checksums.  Returns (u8[STRIDE], len)."""
    f = np.zeros(STRIDE, np.uint8)
    f[0:6], f[6:12] = rcv[6:12], rcv[0:6]
    f[12:14] = (0x08, 0x00)
    f[14] = 0x45
    f[16:18] = S.port_bytes(20 + 8 + qlen)
    f[22], f[23] = 64, 1
    f[26:30], f[30:34] = rcv[30:34], rcv[26:30]
    f[24:26] = S.ip_checksum(f[None, 14:34])[0]
    f[34], f[35] = typ, code
    if mtu:
        f[40:42] = S.port_bytes(mtu)
    if typ == 12:
        f[38] = 9  # pointer
    f[42:42 + qlen] = rcv[14:14 + qlen]
    c = ~inet_csum(f[34:42 + qlen]) & 0xFFFF
    f[36:38] = (c >> 8, c & 0xFF)
    return f, 42 + qlen


def random_error(r, rcv):
    typ = int(r.choice(ERR_TYPES))
    code = int(r.integers(0, 16)) if typ == 3 else int(r.integers(0, 2))
    return sub_error(rcv, int(r.choice([28, 48, 50])), typ, code, 1492 if (typ == 3 and code == 4) else 0)


def not_translatable(r, rcv, j):
    """An error frame of one of the kinds the rule must leave to today's path."""
    f, l = random_error(r, rcv)
    k = j % 11
    if k == 0:  # a flow that never existed: another quoted port (or ICMP id)
        f[64 if f[51] != 1 else 66] ^= 0x5A
    elif k == 1:  # the quote is not addressed to the error's source
        f[61] ^= 0x01
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
    elif k == 6:  # short quote
        l = 42 + int(r.integers(8, 24))
    elif k == 7:  # echo request / reply, source quench / redirect: not error frames
        f[34] = [0, 8, 4, 5][(j // 11) % 4]
    elif k == 8:  # a public source
        f[26:30] = S.ip_bytes(0x08080909)
    elif k == 9:  # a quoted source port no flow has
        f[62 if f[51] != 1 else 67] ^= 0x21
    else:  # a repeat: the same untranslatable error twice (the second hits the echo-keyed session of the first)
        f[61] ^= 0x02
    return f, l


def base_script(prog, seed=0x1CE6, n_subs=N_SUBS, per=6, buckets="open"):
    """Maps, one nat44_egress batch of the flows, one nat44_ingress batch of their replies.  Returns (script, original
    frames, egress step tag, ingress step tag).  buckets: "open" (unlimited), "tight" (rate-limited, small bursts)."""
    r = np.random.default_rng(seed)
    sc = harness.Script("nat_icmp_egress")
    keys, v = S.bindings(n_subs)
    sc.update("subscriber_bindings", keys, v)
    cfg = np.zeros(1, L.antispoof_config)
    cfg["default_mode"], cfg["log_violations"] = 1, 1
    sc.update1("antispoof_config", np.uint32(0), cfg)
    scenarios.nat_maps(sc, n_subs - 1, 64, 0x0F)
    qk, qv = S.qos_buckets(n_subs)
    if buckets == "open":
        qv["rate_bps"] = 0
    else:
        qv["rate_bps"] = np.where(np.arange(n_subs) % 2, 8_000, 0)
        qv["burst_bytes"] = np.where(np.arange(n_subs) % 2, 600, 20000)
        qv["tokens"] = qv["burst_bytes"]
    sc.update("qos_ingress", qk, qv)
    orig = flows(r, n_subs, per)
    sc.run("nat44_egress", scenarios.fixed(orig), np.full(len(orig), 64, np.uint32), T0)
    eg = f"s{len(sc.steps) - 1:03d}"

    def replies(res):
        snat = res[eg + "_frames"].reshape(-1, 64)
        rep = np.stack([reply_of(f) for f in snat])
        return {"arena": rep.reshape(-1).copy(), "lens": np.full(len(rep), 64, np.uint32), "now_ns": T0 + 10**8,
                "stride": 64}

    sc.run_from("nat44_ingress", replies)
    ing = f"s{len(sc.steps) - 1:03d}"
    return sc, orig, eg, ing


def received(res, ing):
    """The replies as the subscribers received them (nat44_ingress's output)."""
    return res[ing + "_frames"].reshape(-1, 64)


def mixed(res, orig, ing, seed, now, frame_clock=False, errors=True, bad=True, copies=2, new_flows=True):
    """A batch of the subscribers' ordinary frames (their flows again, and new flows) interleaved with errors quoting
    the replies they received, the untranslatable kinds, and the ordering case: an error about a flow the same batch
    creates, placed after the flow's first frame (translates) or before it (today's path)."""
    r = np.random.default_rng(seed)
    rcv = received(res, ing)
    rows, lens = [], []
    for _ in range(copies):
        for f in orig:
            g = np.zeros(STRIDE, np.uint8)
            g[:64] = f
            rows.append(g)
            lens.append(64)
        if errors:
            for j, f in enumerate(rcv):
                if f[30] == 100:  # delivered (DNATed) to a subscriber
                    rows.append(random_error(r, f)[0])
                    lens.append(int(rows[-1][16]) * 256 + int(rows[-1][17]) + 14)
    if bad:
        for j in range(len(rcv)):
            f, l = not_translatable(r, rcv[j] if rcv[j][30] == 100 else reply_of(orig[j]), j)
            rows.append(f)
            lens.append(l)
            if j % 11 == 10:  # the repeat
                rows.append(f.copy())
                lens.append(l)
    order = list(r.permutation(len(rows)))
    a = [rows[i] for i in order]
    ln = [lens[i] for i in order]
    if new_flows:  # the ordering case
        fresh = flows(r, N_SUBS - 1, 2, sport0=30000 + seed * 64)
        for k, f in enumerate(fresh):
            g = np.zeros(STRIDE, np.uint8)
            g[:64] = f
            e, el = random_error(r, reply_of(f))
            at = int(r.integers(0, len(a) + 1))
            if k % 2:  # the error first: the flow does not exist yet
                a[at:at] = [e, g]
                ln[at:at] = [el, 64]
            else:
                a[at:at] = [g, e]
                ln[at:at] = [64, el]
    arena = np.stack(a)
    lens = np.array(ln, np.uint32)
    d = {"arena": arena.reshape(-1).copy(), "lens": lens, "now_ns": now, "stride": STRIDE}
    if frame_clock:
        d["now_v"] = (now + np.sort(r.integers(0, 500_000, len(lens)))).astype(np.uint64)
    return d


def script_with(prog, frame_clock=False, buckets="open", **kw):
    sc, orig, eg, ing = base_script(prog, buckets=buckets, **kw)
    sc.run_from(prog, lambda res: mixed(res, orig, ing, 1, T0 + 10**9, frame_clock))
    sc.run_from(prog, lambda res: mixed(res, orig, ing, 2, T0 + 2 * 10**9, frame_clock))
    return sc, orig, eg, ing


class EgressBackend(harness.GpuBackend):
    def __init__(self, pinned=False, on=True, setup=None, **opts):
        super().__init__(pinned=pinned, **opts)
        if on:
            self.dp.nat_icmp_errors_egress_enable(True)
        if setup:
            setup(self.dp)


def check(sc, kind, pinned, what, setup=None, **opts):
    ora = RuleOracle(kind)
    want = harness.run_script(ora, sc)
    be = EgressBackend(pinned, setup=setup, **opts)
    try:
        got = harness.run_script(be, sc)
    finally:
        be.close()
    harness.compare(want, got, f"{what}: {kind} oracle with the rule restated vs gpu")
    return want, ora


# ---------------------------------------------------------------------------
# 1. the restatement, checked without a GPU; and today's behaviour
# ---------------------------------------------------------------------------
def test_restatement_quotes_the_remotes_frame(ora_kind):
    """A translated error quotes the remote's original frame (IPv4 header and 8 L4 bytes, up to a checksum 0x0000 /
    0xFFFF), leaves from the subscriber's public address, and has valid outer, quoted and ICMP checksums."""
    _need(ora_kind)
    sc, orig, eg, ing = script_with("nat44_egress")
    ora = RuleOracle(ora_kind)
    res = harness.run_script(ora, sc)
    snat = res[eg + "_frames"].reshape(-1, 64)
    remote = {}  # the remote's original frames (the replies before nat44_ingress), by their quoted identity
    for f in snat:
        g = reply_of(f)
        remote[bytes(g[26:34]) + bytes(g[34:38] if g[23] != 1 else g[38:40]) + bytes([g[23]])] = g
    pub_of = {bytes(f[6:12]): bytes(f[26:30]) for f in snat}
    runs = [k for k in sorted(res) if k.endswith("_frames")][2:]
    assert len(runs) == len(ora.translated) - 1 == 2  # (the first: the batch that made the flows)
    total = 0
    for k, done in zip(runs, ora.translated[1:]):
        a = res[k].reshape(-1, STRIDE)
        lens = res[k.replace("_frames", "_len")]
        total += len(done)
        for f in a:  # ... and the flows this batch created (the ordering case)
            if f[26] == 203 and not is_error_frame(f, 64):
                g = reply_of(f[:64])
                remote.setdefault(bytes(g[26:34]) + bytes(g[34:38] if g[23] != 1 else g[38:40]) + bytes([g[23]]), g)
        for i in done:
            f = a[i]
            ip = int(f[51])
            key = bytes(f[54:62]) + bytes(f[62:66] if ip != 1 else f[66:68]) + bytes([ip])
            want = remote.get(key)
            assert want is not None, f"{k} frame {i}: quotes no remote frame"
            q, w = f[42:70].copy(), want[14:42].copy()
            for c in (10, {17: 26, 1: 22}.get(ip)):  # the quoted IPv4 checksum, and the UDP / ICMP checksum
                if c is not None and {rd16(q, c), rd16(w, c)} == {0, 0xFFFF}:
                    q[c:c + 2] = w[c:c + 2]
            assert np.array_equal(q, w), f"{k} frame {i}: quote differs from the remote's frame"
            assert bytes(f[26:30]) == pub_of[bytes(f[6:12])], f"{k} frame {i}: not from the public address"
            assert inet_csum(f[14:34]) == 0xFFFF and inet_csum(f[42:62]) == 0xFFFF
            assert inet_csum(f[34:int(lens[i])]) == 0xFFFF, f"{k} frame {i}: ICMP checksum"
    assert total > 150, total


def test_today_corrupts_and_creates(ora_kind):
    """With the switch off, nat44_egress keys a subscriber's error by bytes 4-5: it overwrites them with a NAT port and
    creates an ICMP session (and a SESSION_CREATE record) for a flow that never existed; the quote keeps the private
    address."""
    _need(ora_kind)
    sc, orig, eg, ing = base_script("nat44_egress")

    def one(res):
        f, l = sub_error(received(res, ing)[1], 28, 12, 0)  # a Parameter Problem, pointer 9, about a UDP reply
        return {"arena": f.copy(), "lens": np.array([l], np.uint32), "now_ns": T0 + 10**9, "stride": STRIDE}

    sc.run_from("nat44_egress", one)
    o = harness.OracleBackend(ora_kind)
    res = harness.run_script(o, sc)
    f = res[sorted(k for k in res if k.endswith("_frames"))[-1]]
    assert f[38] != 9 or f[39] != 0  # the pointer is gone
    assert f[58] == 100  # the quote still names the subscriber's private address
    k = res["tk_nat_sessions"]
    echo = (orig[:(N_SUBS - 1) * 6, 23] == 1).sum()  # the echo flows of the subscribers with a NAT block
    assert (k[:, 12] == 1).sum() == echo + 1  # one ICMP session more
    assert res["ev_nat_log_rb"].shape[0] == len(k)  # a SESSION_CREATE record for each, the bogus one included


# ---------------------------------------------------------------------------
# 2. against the GPU
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("clock", ["batch", "frame"])
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("prog", PROGS)
def test_mixed_batches(prog, pinned, clock, ora_kind):
    _need(ora_kind)
    buckets = "tight" if prog != "nat44_egress" else "open"
    sc, _, _, _ = script_with(prog, frame_clock=clock == "frame", buckets=buckets)
    want, ora = check(sc, ora_kind, pinned, f"{prog} mixed ({FEED_IDS[FEEDS.index(pinned)]}, {clock} clock)")
    assert sum(len(t) for t in ora.translated) > 100
    if prog == "pipeline_tc":
        v = [want[k] for k in sorted(want) if k.endswith("_verdict")][-2:]
        assert all((x == L.TC_ACT_SHOT).any() for x in v)  # the bucket dropped some frames


@pytest.mark.gpu
@pytest.mark.parametrize("prog", PROGS)
def test_ordering(prog, ora_kind):
    """An error about a flow the same batch creates translates when the flow's frame comes first, and takes today's
    path when it comes later."""
    _need(ora_kind)
    sc, orig, eg, ing = base_script(prog)

    def batch(res):
        r = np.random.default_rng(9)
        fresh = flows(r, N_SUBS - 1, 2, sport0=31000)
        rows, lens = [], []
        for k, f in enumerate(fresh):
            g = np.zeros(STRIDE, np.uint8)
            g[:64] = f
            e, el = random_error(r, reply_of(f))
            pair = [(g, 64), (e, el)] if k % 2 == 0 else [(e, el), (g, 64)]
            for x, l in pair:
                rows.append(x)
                lens.append(l)
        return {"arena": np.stack(rows).reshape(-1).copy(), "lens": np.array(lens, np.uint32), "now_ns": T0 + 10**9,
                "stride": STRIDE}

    sc.run_from(prog, batch)
    _, ora = check(sc, ora_kind, False, f"{prog} ordering")
    done = ora.translated[-1]
    assert len(done) == N_SUBS - 1 and all(i % 4 == 1 for i in done), done


@pytest.mark.gpu
@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
def test_lengths_and_rings(pinned, ora_kind):
    """Every length from 34 to 100 bytes, and the same errors through a 64-byte header-split ring, where every error
    takes today's path."""
    _need(ora_kind)
    sc, orig, eg, ing = base_script("nat44_egress")

    def lengths(res, stride):
        r = np.random.default_rng(3)
        rcv = received(res, ing)
        rows, lens = [], []
        for l in range(34, 101):
            for f in rcv[r.permutation(len(rcv))[:4]]:
                e, _ = random_error(r, f)
                rows.append(e[:stride])
                lens.append(l)
        return {"arena": np.stack(rows).reshape(-1).copy(), "lens": np.array(lens, np.uint32), "now_ns": T0 + 10**9,
                "stride": stride}

    sc.run_from("nat44_egress", lambda res: lengths(res, STRIDE))
    sc.run_from("nat44_egress", lambda res: lengths(res, 64))
    _, ora = check(sc, ora_kind, pinned, f"lengths ({FEED_IDS[FEEDS.index(pinned)]})")
    assert len(ora.translated[1]) > 60 and len(ora.translated[2]) == 0  # ([0]: the batch that made the flows)


@pytest.mark.gpu
def test_zero_copy_chunk_edges(ora_kind):
    """Errors on both sides of the 2^18-frame chunk edges of the pinned feed."""
    _need(ora_kind)
    sc, orig, eg, ing = base_script("nat44_egress")

    def big(res, n, seed):
        r = np.random.default_rng(seed)
        rcv = received(res, ing)
        pick = r.integers(0, len(orig), n)
        a = np.zeros((n, STRIDE), np.uint8)
        a[:, :64] = orig[pick]
        lens = np.full(n, 64, np.uint32)
        edge = np.zeros(n, bool)
        for e in range(1 << 18, n, 1 << 18):
            edge[max(0, e - 20):e + 20] = True
        for i in np.nonzero(edge)[0]:
            a[i], lens[i] = random_error(r, rcv[pick[i]])
        return {"arena": a.reshape(-1).copy(), "lens": lens, "now_ns": T0 + seed * 10**9, "stride": STRIDE}

    sc.run_from("nat44_egress", lambda res: big(res, (1 << 18) + 77, 1))
    sc.run_from("nat44_egress", lambda res: big(res, (1 << 19) + 5, 2))
    _, ora = check(sc, ora_kind, True, "chunk edges", max_batch=1 << 20)
    assert ora.snat > 60


@pytest.mark.gpu
@pytest.mark.parametrize("combo", ["acct", "qos_ipv6", "antispoof_ipv6", "all"])
@pytest.mark.parametrize("prog", ["pipeline_up", "pipeline_tc"])
def test_combinations(prog, combo, ora_kind):
    """The switch with accounting, bng_qos_ipv6_enable and bng_antispoof_ipv6_prefixes_enable."""
    _need(ora_kind)
    sc, _, _, _ = script_with(prog, buckets="tight")

    def setup(dp):
        if combo in ("acct", "all"):
            dp.acct_enable(prog)
        if combo in ("qos_ipv6", "all"):
            dp.qos_ipv6_enable(True)
        if combo in ("antispoof_ipv6", "all"):
            dp.antispoof_ipv6_prefixes_enable(True)

    check(sc, ora_kind, False, f"{prog} with {combo}", setup=setup)


@pytest.mark.gpu
def test_both_directions(ora_kind):
    """Both switches on: nat44_ingress translates a remote's error inbound (bng_nat_icmp_errors_enable) and
    nat44_egress a subscriber's error outbound in the same run of the script."""
    _need(ora_kind)
    import test_gpu_nat_icmp as IN
    sc, orig, eg, ing = base_script("nat44_egress")

    def inbound(res):
        snat = res[eg + "_frames"].reshape(-1, 64)
        r = np.random.default_rng(4)
        rows, lens = [], []
        for f in snat:
            e, l = IN.random_error(r, f)
            rows.append(e)
            lens.append(l)
        return {"arena": np.stack(rows).reshape(-1).copy(), "lens": np.array(lens, np.uint32), "now_ns": T0 + 10**9,
                "stride": STRIDE}

    sc.run_from("nat44_ingress", inbound)
    sc.run_from("nat44_egress", lambda res: mixed(res, orig, ing, 5, T0 + 2 * 10**9, bad=False, new_flows=False))

    class Both(RuleOracle):
        def __init__(self, kind):
            super().__init__(kind)
            self.inb = IN.RuleOracle(kind)
            self.inb.o = self.o

        def run(self, prog, arena, lens, now, off16, stride, prio, now_v=None):
            if prog == "nat44_ingress":
                return self.inb.run(prog, arena, lens, now, off16, stride, prio, now_v)
            return super().run(prog, arena, lens, now, off16, stride, prio, now_v)

        def stats(self, m):
            s = super().stats(m)
            if m == "nat_stats_map":
                s = s.copy()
                s[list(L.nat_stats.names).index("packets_dnat")] += self.inb.dnat
                s[list(L.nat_stats.names).index("packets_passed")] += self.inb.passed
            return s

    ora = Both(ora_kind)
    want = harness.run_script(ora, sc)
    be = EgressBackend(False, setup=lambda dp: dp.nat_icmp_errors_enable(True))
    try:
        got = harness.run_script(be, sc)
    finally:
        be.close()
    harness.compare(want, got, "both switches: oracle with both rules restated vs gpu")
    assert ora.inb.dnat > 20 and ora.snat > 20


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
@pytest.mark.parametrize("prog", PROGS)
def test_off_is_today(prog, ora_kind):
    _need(ora_kind)
    sc, _, _, _ = script_with(prog)
    today = harness.run_script(harness.OracleBackend(ora_kind), sc)  # errors keyed by bytes 4-5, as ever
    never = _observe(sc, lambda dp: None)
    harness.compare(today, never[2], f"{prog} never set: oracle vs gpu")
    assert not any("icmperr" in k for k in never[1])

    def on_off(dp):
        dp.nat_icmp_errors_egress_enable(True)
        dp.nat_icmp_errors_egress_enable(False)

    again = _observe(sc, on_off)
    harness.compare(today, again[2], f"{prog} on, then off: oracle vs gpu")
    assert again[:2] == never[:2]
    # with no error frames in the batches, "on" computes what the oracle does
    quiet, orig, eg, ing = base_script(prog)
    quiet.run_from(prog, lambda res: mixed(res, orig, ing, 5, T0 + 10**9, errors=False, bad=False, new_flows=False))
    on = _observe(quiet, lambda dp: dp.nat_icmp_errors_egress_enable(True))
    harness.compare(harness.run_script(harness.OracleBackend(ora_kind), quiet), on[2], f"{prog} on, no errors")
    assert any(k.endswith(", icmperr>)") and "k_resolve" in k for k in on[1])
    assert any(k.endswith("icmperr>)") and "k_pipe_classify" in k for k in on[1])


# ---------------------------------------------------------------------------
# 4. attribution: accounting, idle stamps and interception see the frame as it entered
# ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_attribution(ora_kind):
    _need(ora_kind)
    prog = "pipeline_up"
    sc, orig, eg, ing = base_script(prog)
    sc.run_from(prog, lambda res: mixed(res, orig, ing, 7, T0 + 10**9, copies=1, new_flows=False))
    ora = RuleOracle(ora_kind)
    want = harness.run_script(ora, sc)
    subs = S.ip_bytes(S.sub_ip(np.arange(N_SUBS)))
    sub_words = subs.copy().view("<u4").reshape(-1)
    tag = sorted(k for k in want if k.endswith("_frames"))[-1][:4]
    inp = sc.steps[-1][2](want)  # the batch as it entered
    a_in = inp["arena"].reshape(-1, STRIDE)
    be = EgressBackend(False)
    try:
        dp = be.dp
        dp.acct_enable(prog)
        dp.idle_enable(prog)
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
    done = set(ora.translated[-1].tolist())
    assert len(done) > 20
    v = want[tag + "_verdict"]
    lens = want[tag + "_len"]
    src = a_in[:, 26:30].copy().view("<u4").reshape(-1)
    ok4 = (a_in[:, 12] == 0x08) & (a_in[:, 13] == 0x00)
    for j, w in enumerate(sub_words[:N_SUBS - 1]):
        mine = np.nonzero((src == w) & ok4 & (v != L.TC_ACT_SHOT))[0]
        assert acct[j]["up_packets"] == len(mine) and acct[j]["up_bytes"] == int(lens[mine].sum()), j
        assert any(i in done for i in mine), f"subscriber {j} sent no translated error"
        assert idle[j]["up_ns"] == T0 + 10**9
    # captured as the subscriber sent it: every capture of this batch holds the frame as it entered
    last = hdr["dir"] == 0
    if "batch" in hdr.dtype.names:
        last &= hdr["batch"] == hdr["batch"][last].max()
    caught = [(int(h["frame"]), d) for h, d, x in zip(hdr, data, last) if x]
    assert any(i in done for i, _ in caught)
    for i, d in caught:
        assert np.array_equal(d, a_in[i, :len(d)]), i


# ---------------------------------------------------------------------------
# 5. the interface (no GPU)
# ---------------------------------------------------------------------------
def test_header_declares_the_call():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "bng_b200.h")).read(), flags=re.S)
    assert re.search(r"int\s+bng_nat_icmp_errors_egress_enable\s*\(\s*bng_ctx\s*\*\s*ctx\s*,\s*int\s+on\s*\)\s*;", src)


def test_binding_exposes_the_call():
    assert "bng_nat_icmp_errors_egress_enable" in D.EXPORTED_SYMBOLS
    assert callable(Dataplane.nat_icmp_errors_egress_enable)


def test_null_context_is_einval():
    lib = D.load_library()
    assert lib.bng_nat_icmp_errors_egress_enable(None, 1) == -errno.EINVAL
    assert lib.bng_nat_icmp_errors_egress_enable(None, 0) == -errno.EINVAL
