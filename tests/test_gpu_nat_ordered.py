"""New NAT flows created in the resolve kernel's ordered phase, at the edges of the port block, against the oracle.

Most new flows do not go through the sequential nat44_egress of the ordered phase: nat_chunk_coop
(bng_b200/csrc/progs.cuh) parses, probes, allocates and commits up to 32 new flows of one subscriber at once, as long
as they provably do not interact, and sends the first frame that might to the sequential code.  Its clash rules each
restate a piece of allocate_port_from_block() and get_eim_mapping() (bpf/nat44.c:408-528): the counter at 0 or
outside the block, a counter that wraps, candidates taken by EIM keys that exist or that an earlier flow creates,
repeated 5-tuples, endpoints and nat_reverse keys.

Every case below is one small script of hand-built port blocks, pre-installed EIM mappings and new flows, arranged so
that a 32-frame chunk meets one edge.  It runs on the oracle and on the GPU (nat44_egress, pipeline_up and pipeline_tc;
EIM on and off; one clock per batch and one per frame; pageable and device-resident feeds, pinned for nat44_egress),
and the two must agree bit for bit.  Each case also says which paths it must take: the dataplane's ST_NAT_COOP and
ST_NAT_SEQ counters are read before and after, so a case whose cooperative or sequential branch did not run fails
instead of quietly testing something else.  A seeded differential draws blocks, counters and mappings from the same
edges for a few dozen subscribers at a time.

The tests without the gpu mark run every case on the oracle alone and check the reference outcome it claims to
construct (a port-0 candidate is exhaustion, an exactly used block leaves the counter at port_start, ...), so the case
builders stay honest on every CPU run."""
from __future__ import annotations

from typing import Callable, NamedTuple

import numpy as np
import pytest

import harness
from bng_b200 import layouts as L
from bng_b200 import synth as S

GW_MAC = 0x02FFFFFFFFFE
PUB0 = 0xCB007100      # subscriber i translates to PUB0 + i (one address each: no flows of two subscribers interact)
DST0 = 0x08080800      # destination k is DST0 + k
NATF_EIM, NATF_HAIRPIN, NATF_ALG = 0x01, 0x04, 0x18
ST_NAT_COOP, ST_NAT_SEQ, ST_LRU_EVICT = 37, 38, 39  # bng_b200/csrc/common.cuh
NS = {n: i for i, n in enumerate(L.nat_stats.names)}
EV_CREATE, EV_EXHAUST, EV_ALG = 1, 5, 7
PROGS = ["nat44_egress", "pipeline_up", "pipeline_tc"]
CLOCKS = ["batch", "frame"]
T0 = 10**9


def _need(kind):
    if kind == "none":
        pytest.fail("no oracle library present on this box")


# ---------------------------------------------------------------------------
# case description
# ---------------------------------------------------------------------------
class F(NamedTuple):
    """One frame: subscriber, source port (host order; the ICMP echo id for proto 1), destination index, destination
    port, protocol and a kind: "" a plain frame, "alg" (to the FTP control port), "gre" (not translatable), "opts"
    (IPv4 options), "short" (TCP header cut short), "hairpin" (to subscriber 0's public address), "icmperr" (an ICMP
    Destination Unreachable that quotes no flow)."""
    sub: int
    sport: int
    dst: int = 0
    dport: int = 443
    proto: int = 6
    kind: str = ""


class Case(NamedTuple):
    name: str
    blocks: list          # (port_start, port_end, next_port) per subscriber
    batches: list         # list of lists of F
    path: Callable        # eim -> "coop" (cooperative only) or "both" (both paths run)
    check: Callable       # (oracle results, eim) -> None: the reference outcome the case constructs
    pre: list = []        # pre-installed eim_table keys (sub, internal_port as stored, proto[, external_port])
    opts: dict = {}       # Dataplane sizes (the capacity case)
    icmperr: bool = False  # bng_nat_icmp_errors_egress_enable


def le(port):
    """The source port whose network-order bytes, loaded little-endian, read as `port` (an EIM key that
    allocate_port_from_block() finds when it probes candidate `port`, bpf/nat44.c:450-455)."""
    return ((port & 0xFF) << 8) | (port >> 8)


def new_flows(sub, n, sport0=40000, dst=0, proto=6):
    return [F(sub, sport0 + i, dst, 443, proto) for i in range(n)]


# ---------------------------------------------------------------------------
# reading the oracle's results
# ---------------------------------------------------------------------------
def stat(res, name):
    return int(res["st_nat_stats_map"][NS[name]])


def sessions(res):
    """{(subscriber, source port, destination index, destination port, protocol): nat port (host order)}"""
    k = res["tk_nat_sessions"].view(L.nat_key).reshape(-1)
    v = res["tv_nat_sessions"].view(L.nat_session).reshape(-1)
    out = {}
    for kk, vv in zip(k, v):
        src = int.from_bytes(bytes(kk["src_ip"]), "big") - int(S.sub_ip(0))
        dst = int.from_bytes(bytes(kk["dst_ip"]), "big") - DST0
        out[(src, int.from_bytes(bytes(kk["src_port"]), "big"), dst, int.from_bytes(bytes(kk["dst_port"]), "big"),
             int(kk["protocol"]))] = int.from_bytes(bytes(vv["nat_port"]), "big")
    return out


def next_ports(res):
    """next_port per subscriber index"""
    k, v = res["tk_subscriber_nat"], res["tv_subscriber_nat"].view(L.subscriber_nat).reshape(-1)
    return {int.from_bytes(bytes(kk), "big") - int(S.sub_ip(0)): int(vv["block"]["next_port"]) for kk, vv in zip(k, v)}


def events(res, kind):
    ev = res["ev_nat_log_rb"]
    if ev.shape[0] == 0 or ev.shape[1] != L.nat_log_entry.itemsize:
        return np.zeros(0, L.nat_log_entry)
    e = np.ascontiguousarray(ev).view(L.nat_log_entry).reshape(-1)
    return e[e["event_type"] == kind]


def verdicts(res):
    return np.concatenate([res[k] for k in sorted(res) if k.endswith("_verdict")])


def key(f: F):
    return (f.sub, f.sport, f.dst, f.dport, f.proto)


def ports(res, flows):
    s = sessions(res)
    return [s.get(key(f)) for f in flows]


def no_port_zero(res):
    assert 0 not in sessions(res).values(), "a session translated to port 0"
    assert not (events(res, EV_CREATE)["public_port"] == 0).all(axis=1).any(), "SESSION_CREATE with port 0"


def exhausted(res, eim, n=1):
    """n port-0 candidates: each is port exhaustion; without EIM the frame is dropped and logged, with EIM it falls
    back to a port without a mapping (bpf/nat44.c:501-504, :694-705)."""
    assert stat(res, "port_exhaustion") == n
    no_port_zero(res)
    if eim:
        assert stat(res, "packets_dropped") == 0 and len(events(res, EV_EXHAUST)) == 0
    else:
        assert stat(res, "packets_dropped") == n and len(events(res, EV_EXHAUST)) == n
        assert (verdicts(res) == L.TC_ACT_SHOT).sum() == n


# ---------------------------------------------------------------------------
# the constructed cases
# ---------------------------------------------------------------------------
def _both(eim):
    return "both"


def _coop(eim):
    return "coop"


def _port0_start0():
    fl = new_flows(0, 6)

    def check(res, eim):
        exhausted(res, eim)
        assert ports(res, fl) == ([1, 2, 3, 4, 5, 6] if eim else [None, 1, 2, 3, 4, 5])
    return Case("port0_start0", [(0, 7, 0)], [fl], _both, check)


def _port0_next0():
    fl = new_flows(0, 5)

    def check(res, eim):
        exhausted(res, eim)
        # the counter runs on from 0: the ports below the block are handed out
        assert ports(res, fl) == ([1, 2, 3, 4, 5] if eim else [None, 1, 2, 3, 4])
    return Case("port0_next0", [(1024, 1055, 0)], [fl], _both, check)


def _port0_wrap():
    # [0, 7] from 3: five flows end the block exactly, a repeated 5-tuple ends the cooperative prefix, and the next
    # new flow meets the counter at 0 on the cooperative path
    fl = new_flows(0, 5)
    more = new_flows(0, 4, sport0=41000)
    b1 = fl + [fl[0]] + more

    def check(res, eim):
        exhausted(res, eim)
        assert ports(res, fl) == [3, 4, 5, 6, 7]
        assert ports(res, more) == ([1, 2, 3, 4] if eim else [None, 1, 2, 3])
    return Case("port0_wrap", [(0, 7, 3)], [b1], _both, check)


def _port0_next_batch():
    # the first batch uses [0, 7] up exactly from 4; the second starts at 0
    fl, more = new_flows(0, 4), new_flows(0, 4, sport0=41000)

    def check(res, eim):
        exhausted(res, eim)
        assert next_ports(res)[0] == (5 if eim else 4)
    return Case("port0_next_batch", [(0, 7, 4)], [fl, more], _both, check)


def _below_start():
    fl = new_flows(0, 8)

    def check(res, eim):
        assert ports(res, fl) == list(range(1000, 1008)) and next_ports(res)[0] == 1008
    return Case("next_below_start", [(1024, 1055, 1000)], [fl], _coop, check)


def _past_end():
    fl = new_flows(0, 6)

    def check(res, eim):
        # a candidate past the end is replaced by port_start, and so is the counter: port_start comes out twice
        assert ports(res, fl) == [1024, 1024, 1025, 1026, 1027, 1028]
    return Case("next_past_end", [(1024, 1031, 2000)], [fl], _both, check)


def _next_ffff():
    fl = new_flows(0, 4)
    fl2 = new_flows(1, 4)

    def check(res, eim):
        assert ports(res, fl) == [1024, 1024, 1025, 1026]
        assert ports(res, fl2) == [65535, 65528, 65529, 65530]  # a block ending at 65535 hands 0xFFFF out, then wraps
    return Case("next_ffff", [(1024, 1031, 0xFFFF), (65528, 65535, 0xFFFF)], [fl + fl2], _both, check)


def _next_10000():
    fl = new_flows(0, 4)
    fl2 = new_flows(1, 4)

    def check(res, eim):
        # (u16)0x10000 is 0: exhaustion, once per subscriber, then the counter is back at port_start
        exhausted(res, eim, 2)
        assert ports(res, fl) == ([1024, 1025, 1026, 1027] if eim else [None, 1024, 1025, 1026])
        assert ports(res, fl2) == ([65528, 65529, 65530, 65531] if eim else [None, 65528, 65529, 65530])
    return Case("next_10000", [(1024, 1031, 0x10000), (65528, 65535, 0x10000)], [fl + fl2], _both, check)


def _next_1ffff():
    fl = new_flows(0, 4)
    fl2 = new_flows(1, 4)

    def check(res, eim):
        assert ports(res, fl) == [1024, 1024, 1025, 1026]  # (u16)0x1FFFF = 0xFFFF
        assert ports(res, fl2) == [65535, 65528, 65529, 65530]
    return Case("next_1ffff", [(1024, 1031, 0x1FFFF), (65528, 65535, 0x1FFFF)], [fl + fl2], _both, check)


def _end_below_start():
    # [2000, 1990] from 1985: 1985..1990, then port_start over and over
    fl = [F(0, 40000 + i, i, 443, 6) for i in range(10)]

    def check(res, eim):
        assert ports(res, fl) == list(range(1985, 1991)) + [2000] * 4 and next_ports(res)[0] == 2000
    return Case("end_below_start", [(2000, 1990, 1985)], [fl], _both, check)


def _end_65535():
    fl = new_flows(0, 10)
    fl2 = new_flows(1, 6)

    def check(res, eim):
        assert ports(res, fl) == list(range(65530, 65536)) + [65000, 65001, 65002, 65003]
        exhausted(res, eim)  # [0, 65535] wraps to 0
        assert ports(res, fl2)[:3] == [65533, 65534, 65535]
    return Case("end_65535", [(65000, 65535, 65530), (0, 65535, 65533)], [fl + fl2], _both, check)


def _block_exact():
    fl = new_flows(0, 8)
    fl2 = new_flows(1, 32, proto=17)

    def check(res, eim):
        assert ports(res, fl) == list(range(1024, 1032)) and ports(res, fl2) == list(range(2048, 2080))
        assert next_ports(res) == {0: 1024, 1: 2048}
    return Case("block_exact", [(1024, 1031, 1024), (2048, 2079, 2048)], [fl, fl2], _coop, check)


def _block_plus_one():
    fl = [F(0, 40000 + i, 0, 443 + (i == 8), 6) for i in range(9)]

    def check(res, eim):
        assert ports(res, fl) == list(range(1024, 1032)) + [1024] and next_ports(res)[0] == 1025
    return Case("block_plus_one", [(1024, 1031, 1024)], [fl], _both, check)


def _eim_existing(at):
    # an EIM key of the subscriber that reads as candidate 1024 + at: allocate_port_from_block() skips that port,
    # with EIM on or off
    fl = new_flows(0, 8)

    def check(res, eim):
        assert ports(res, fl) == [p for p in range(1024, 1033) if p != 1024 + at]
    return Case(f"eim_existing_{at}", [(1024, 1055, 1024)], [fl], _both, check, pre=[(0, 1024 + at, 6)])


def _eim_earlier_lane():
    # lane 0's endpoint is the EIM key that candidate 1027 reads as: with EIM on, lane 3 must skip 1027
    fl = [F(0, le(1027), 0)] + new_flows(0, 7)[1:]

    def check(res, eim):
        assert ports(res, fl) == ([1024, 1025, 1026, 1028, 1029, 1030, 1031] if eim else list(range(1024, 1031)))
    return Case("eim_earlier_lane", [(1024, 1055, 1024)], [fl], lambda eim: "both" if eim else "coop", check)


def _repeat_tuple():
    fl = new_flows(0, 4)
    b = fl + [fl[1]] + new_flows(0, 3, sport0=41000)

    def check(res, eim):
        assert len(sessions(res)) == 7 and stat(res, "sessions_created") == 7 and stat(res, "packets_snat") == 8
    return Case("repeat_tuple", [(1024, 1055, 1024)], [b], _both, check)


def _repeat_endpoint():
    fl = [F(0, 40000, 0), F(0, 40001, 0), F(0, 40000, 1), F(0, 40002, 0)]

    def check(res, eim):
        p = ports(res, fl)
        assert (p[0] == p[2]) == eim and stat(res, "eim_hits") == (1 if eim else 0)
    return Case("repeat_endpoint", [(1024, 1055, 1024)], [fl], lambda eim: "both" if eim else "coop", check)


def _shared_reverse():
    # [1024, 1027] used up by four endpoints to destination 0, port 80.  Next batch: a new endpoint to port 443 gets
    # 1024 again (overwriting nothing), and endpoint 40000 to port 443 — with EIM its mapping's 1024 — shares that
    # nat_reverse key: the later frame must own it
    b1 = [F(0, 40000 + i, 0, 80) for i in range(4)]
    b2 = [F(0, 41000, 0, 443), F(0, 40000, 0, 443), F(0, 41001, 0, 443)]

    def check(res, eim):
        rk = res["tk_nat_reverse"].view(L.nat_key).reshape(-1)
        rv = res["tv_nat_reverse"].view(L.nat_key).reshape(-1)
        own = [int.from_bytes(bytes(v["src_port"]), "big") for k, v in zip(rk, rv)
               if int.from_bytes(bytes(k["dst_port"]), "big") == 1024 and int.from_bytes(bytes(k["src_port"]), "big") == 443]
        assert own == [40000 if eim else 41000]
        assert ports(res, b2) == ([1024, 1024, 1025] if eim else [1024, 1025, 1026])
    return Case("shared_reverse", [(1024, 1027, 1024)], [b1, b2], lambda eim: "both" if eim else "coop", check)


def _odd_frames():
    # frames that are not new translatable flows, in the middle of a chunk of new flows: pipeline_tc runs all of them
    # through the cooperative path, which counts their ALG and hairpin statistics
    fl = [F(0, 40000, 0), F(0, 40001, 0, 21, 6, "alg"), F(0, 40002, 0), F(0, 40003, 0, 443, 6, "gre"),
          F(0, 40004, 0, 443, 6, "opts"), F(0, 40005, 0, 443, 6, "short"), F(0, 40006, 0, 443, 6, "hairpin"),
          F(0, 40007, 0, 443, 17, "opts"), F(0, 40008, 1)]

    def check(res, eim):
        assert stat(res, "alg_triggers") == 1 and len(events(res, EV_ALG)) == 1
        assert stat(res, "packets_hairpin") == 1 and stat(res, "sessions_created") == 6
        assert next_ports(res)[0] == 1030
    return Case("odd_frames", [(1024, 1055, 1024)], [fl], _coop, check)


def _icmp_error():
    fl = new_flows(0, 3) + [F(0, 777, 2, 0, 1, "icmperr")] + new_flows(0, 3, sport0=41000)

    def check(res, eim):
        assert ports(res, fl) == list(range(1024, 1031))
    return Case("icmp_error", [(1024, 1055, 1024)], [fl], _both, check, icmperr=True)


def _capacity():
    # room for exactly the 32 sessions, nat_reverse entries and EIM mappings the chunk creates
    fl = [F(0, 40000 + i, i) for i in range(32)]

    def check(res, eim):
        assert len(sessions(res)) == 32 and len(res["tk_nat_reverse"]) == 32
        assert len(res["tk_eim_table"]) == (32 if eim else 0)
    return Case("capacity", [(1024, 1087, 1024)], [fl], _coop, check,
                opts=dict(max_nat_sessions=32, max_eim_mappings=32))


def _fat():
    # 300 new flows of one subscriber (two staging sweeps) with a few repeats; [0, 222] from 32 is used up exactly at
    # the end of the sixth chunk (191 new flows and one repeat), so the seventh starts at 0
    fl = new_flows(0, 300, sport0=30000)
    b = list(fl)
    for at, src in ((100, 3), (250, 200), (290, 7)):
        b.insert(at, fl[src])

    def check(res, eim):
        exhausted(res, eim)
        assert len(sessions(res)) == (300 if eim else 299)
        if not eim:
            assert np.flatnonzero(verdicts(res) == L.TC_ACT_SHOT).tolist() == [192]
    return Case("fat", [(0, 222, 32)], [b], _both, check)


CASES = {c.name: c for c in (
    _port0_start0(), _port0_next0(), _port0_wrap(), _port0_next_batch(), _below_start(), _past_end(), _next_ffff(),
    _next_10000(), _next_1ffff(), _end_below_start(), _end_65535(), _block_exact(), _block_plus_one(),
    _eim_existing(0), _eim_existing(3), _eim_existing(7), _eim_earlier_lane(), _repeat_tuple(), _repeat_endpoint(),
    _shared_reverse(), _odd_frames(), _icmp_error(), _capacity(), _fat())}


# ---------------------------------------------------------------------------
# scripts
# ---------------------------------------------------------------------------
def frames(fl):
    n = len(fl)
    sub = np.array([f.sub for f in fl], np.int64)
    kind = np.array([f.kind for f in fl])
    proto = np.array([47 if f.kind == "gre" else f.proto for f in fl], np.uint32)
    dst = np.array([PUB0 if f.kind == "hairpin" else DST0 + f.dst for f in fl], np.uint32)
    sport = np.array([f.sport for f in fl], np.uint32)
    dport = np.array([f.dport for f in fl], np.uint32)
    lens = np.full(n, 64, np.uint32)
    ck = (0x1000 + np.arange(n)).astype(np.uint32)
    args = (S.sub_mac_key(sub), np.uint64(GW_MAC), S.sub_ip(sub), dst, proto, sport, dport, lens)
    hdr = S.ipv4_headers(*args, l4_check=ck)
    opt = kind == "opts"
    if opt.any():
        hdr[opt] = S.ipv4_headers(*args, l4_check=ck, ihl=6)[opt]
    lens[kind == "short"] = 50
    err = kind == "icmperr"
    hdr[err, 34], hdr[err, 35] = 3, 1
    return hdr.reshape(-1), lens


def setup(sc, blocks, eim, prog, pre=()):
    n = len(blocks)
    idx = np.arange(n)
    v = np.zeros(n, L.subscriber_nat)
    v["block"]["public_ip"] = S.ip_bytes(PUB0 + idx)
    v["block"]["port_start"] = [b[0] for b in blocks]
    v["block"]["port_end"] = [b[1] for b in blocks]
    v["block"]["next_port"] = [b[2] for b in blocks]
    v["block"]["subscriber_id"] = idx + 1
    sc.update("subscriber_nat", S.ip_bytes(S.sub_ip(idx)), v)
    sc.update1("nat_config_map", np.uint32(0), S.nat_config(NATF_HAIRPIN | NATF_ALG | (NATF_EIM if eim else 0), 64))
    sc.update("hairpin_ips", S.ip_bytes(PUB0 + idx), np.ones(n, np.uint8))
    alg = np.zeros(2, L.alg_config)
    alg["port"], alg["protocol"], alg["alg_type"] = [21, 5060], [6, 17], [1, 2]
    sc.update("alg_ports", ((alg["port"].astype(np.uint32) << 16) | alg["protocol"]).astype("<u4"), alg)
    if len(pre):
        k = np.zeros(len(pre), L.eim_key)
        k["internal_ip"] = S.ip_bytes(S.sub_ip(np.array([p[0] for p in pre])))
        k["internal_port"] = [p[1] for p in pre]
        k["protocol"] = [p[2] for p in pre]
        m = np.zeros(len(pre), L.eim_mapping)
        m["external_ip"] = S.ip_bytes(PUB0 + np.array([p[0] for p in pre]))
        m["external_port"] = [p[3] if len(p) > 3 else 60000 + i for i, p in enumerate(pre)]
        m["created"] = m["last_used"] = T0 // 2
        m["ref_count"] = 1
        sc.update("eim_table", k, m)
    if prog.startswith("pipeline"):
        keys, b = S.bindings(n)
        sc.update("subscriber_bindings", keys, b)
        cfg = np.zeros(1, L.antispoof_config)
        cfg["default_mode"] = 1
        sc.update1("antispoof_config", np.uint32(0), cfg)
        # a bucket that passes everything: pipeline_tc then runs every frame's NAT in the ordered phase
        tb = np.zeros(n, L.token_bucket)
        tb["rate_bps"], tb["burst_bytes"] = 10**12, 1 << 30
        tb["tokens"] = tb["burst_bytes"]
        sc.update("qos_ingress", S.ip_bytes(S.sub_ip(idx)), tb)
        sc.update("qos_egress", S.ip_bytes(S.sub_ip(idx)), tb)


def run_batch(sc, prog, fl, b, clock):
    arena, lens = frames(fl)
    now = T0 + b * 10**9
    # per-frame clock: non-decreasing, two frames to a tick
    now_v = None if clock == "batch" else (now + (np.arange(len(fl)) // 2) * 1000).astype(np.uint64)
    sc.run(prog, arena, lens, now, stride=64, now_v=now_v)


def case_script(case: Case, prog: str, eim: bool, clock: str) -> harness.Script:
    sc = harness.Script(f"{case.name}/{prog}/{'eim' if eim else 'noeim'}/{clock}")
    setup(sc, case.blocks, eim, prog, case.pre)
    for b, fl in enumerate(case.batches):
        run_batch(sc, prog, fl, b, clock)
    return sc


# ---------------------------------------------------------------------------
# the dataplane, with the path counters
# ---------------------------------------------------------------------------
class _DevWords:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}


def counters(dp):
    """The dataplane's statistics vector (bng_stats_device_ptr), read from the device."""
    import torch
    dp.sync()
    ptr, n = dp.stats_device_ptr()
    return torch.as_tensor(_DevWords(ptr, n), device="cuda").cpu().numpy().copy()


def run_gpu(sc, feed, opts=None, icmperr=False):
    """(results, coop, seq, evicted) of a script on a fresh dataplane"""
    be = harness.GpuBackend(pinned=feed, **dict(dict(max_subscribers=1 << 10, max_nat_sessions=1 << 12,
                                                     max_eim_mappings=1 << 12, max_batch=1 << 12,
                                                     event_capacity=1 << 12), **(opts or {})))
    try:
        if icmperr:
            be.dp.nat_icmp_errors_egress_enable(True)
        c0 = counters(be.dp)
        res = harness.run_script(be, sc)
        c1 = counters(be.dp)
    finally:
        be.close()
    d = c1 - c0
    return res, int(d[ST_NAT_COOP]), int(d[ST_NAT_SEQ]), int(d[ST_LRU_EVICT])


def check_path(what, path, coop, seq):
    assert coop > 0, f"{what}: no frame took the cooperative path (seq {seq})"
    if path == "coop":
        assert seq == 0, f"{what}: {seq} frames took the sequential path, the case is built for the cooperative one"
    else:
        assert seq > 0, f"{what}: no frame took the sequential path (coop {coop})"


def feeds_of(prog):
    return [False, "device"] + ([True] if prog == "nat44_egress" else [])


# ---------------------------------------------------------------------------
# CPU: the reference outcome each case claims
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("eim", [False, True], ids=["noeim", "eim"])
@pytest.mark.parametrize("name", list(CASES))
def test_case_on_oracle(ora_kind, name, eim):
    _need(ora_kind)
    case = CASES[name]
    be = harness.OracleBackend(ora_kind)
    try:
        res = harness.run_script(be, case_script(case, "nat44_egress", eim, "batch"))
    finally:
        be.close()
    case.check(res, eim)


def test_cases_cover_the_block_edges():
    """Every port-block edge the cooperative path restates has a case, and every case starts a chunk on it."""
    starts = {b[0] for c in CASES.values() for b in c.blocks}
    nexts = {b[2] for c in CASES.values() for b in c.blocks}
    assert {0, 0xFFFF, 0x10000, 0x1FFFF} <= nexts and 0 in starts
    assert any(b[1] < b[0] for c in CASES.values() for b in c.blocks)
    assert any(b[1] == 65535 for c in CASES.values() for b in c.blocks)
    assert max(len(fl) for c in CASES.values() for fl in c.batches) > 256


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("eim", [False, True], ids=["noeim", "eim"])
@pytest.mark.parametrize("prog", PROGS)
@pytest.mark.parametrize("name", list(CASES))
def test_case_gpu(ora_kind, name, prog, eim):
    _need(ora_kind)
    case = CASES[name]
    for clock in CLOCKS:
        sc = case_script(case, prog, eim, clock)
        be = harness.OracleBackend(ora_kind)
        try:
            ref = harness.run_script(be, sc)
        finally:
            be.close()
        for feed in feeds_of(prog):
            what = f"{sc.name}/{feed}"
            got, coop, seq, evicted = run_gpu(sc, feed, case.opts, case.icmperr)
            harness.compare(ref, got, what)
            assert evicted == 0, f"{what}: {evicted} LRU evictions"
            check_path(what, case.path(eim), coop, seq)


# ---------------------------------------------------------------------------
# seeded differential: blocks, counters and EIM keys drawn from the same edges
# ---------------------------------------------------------------------------
N_RAND_SUBS = 40


def random_script(seed, prog, eim):
    r = np.random.Generator(np.random.PCG64(seed))
    n = N_RAND_SUBS
    blocks, pre = [], []
    for s in range(n):
        size = int(r.integers(1, 49))
        start = int(r.choice([0, 1, 1024, 65536 - size, int(r.integers(0, 65536 - size))]))
        end = start + size - 1
        if r.integers(0, 10) == 0:
            end = max(start - int(r.integers(1, 8)), 0)  # port_end < port_start
        nxt = int(r.choice([start, start, 0, max(start - 3, 0), end, end + 1, start + size // 2, 0xFFFF, 0x10000,
                            0x1FFFF]))
        blocks.append((start, end, nxt))
        for c in r.choice(8, int(r.integers(0, 3)), replace=False):  # EIM keys on the next few candidates
            pre.append((s, (nxt + int(c)) & 0xFFFF, int(r.choice([6, 17])), int(r.choice([start, 50000]))))
    sc = harness.Script(f"random/{seed:#x}/{prog}/{'eim' if eim else 'noeim'}")
    setup(sc, blocks, eim, prog, pre)
    for b in range(3):
        fl = []
        for s in range(n):
            nf = int(r.choice([0, 1, 3, 8, 20, 40]))
            cand = [blocks[s][0] + k for k in range(4)]
            sports = [40000 + int(k) for k in range(3)] + [le(p & 0xFFFF) for p in cand]
            for _ in range(nf):
                fl.append(F(s, int(r.choice(sports)), int(r.integers(0, 2)), int(r.choice([443, 80])),
                            int(r.choice([6, 6, 17]))))
        order = r.permutation(len(fl))
        run_batch(sc, prog, [fl[i] for i in order], b, "frame" if b == 1 else "batch")
    return sc


@pytest.mark.gpu
@pytest.mark.parametrize("eim", [False, True], ids=["noeim", "eim"])
@pytest.mark.parametrize("prog", PROGS)
@pytest.mark.parametrize("seed", [0x0D01, 0x0D02, 0x0D03, 0x0D04])
def test_random_gpu(ora_kind, seed, prog, eim):
    _need(ora_kind)
    sc = random_script(seed, prog, eim)
    be = harness.OracleBackend(ora_kind)
    try:
        ref = harness.run_script(be, sc)
    finally:
        be.close()
    got, coop, seq, evicted = run_gpu(sc, "device" if seed & 1 else False)
    harness.compare(ref, got, sc.name)
    assert evicted == 0
    check_path(sc.name, "both", coop, seq)


def test_random_scripts_reach_the_edges(ora_kind):
    """On the oracle: the drawn scripts meet port exhaustion and a wrapped counter for every seed."""
    _need(ora_kind)
    for seed in (0x0D01, 0x0D02, 0x0D03, 0x0D04):
        be = harness.OracleBackend(ora_kind)
        try:
            res = harness.run_script(be, random_script(seed, "nat44_egress", False))
        finally:
            be.close()
        assert stat(res, "port_exhaustion") > 0 and stat(res, "sessions_created") > 100
