"""NAT session counters, last_seen and EIM last_used at their word edges, against the oracle.

The reference counts plain u64s: packets_out++ and bytes_out += skb->len (bpf/nat44.c:679-680, :881 for the _in pair).
The dataplane packs each direction's pair into two u64s (common.cuh, ses_count): the low 32 bits of packets and bytes
advance with one atomic per frame, their high halves only when a low word wraps, and a packet-word wrap spills +1 into
the byte word that is then taken back (ses_count_carry).  The reference overwrites session->last_seen and
mapping->last_used with the frame's clock (:678, :880, :485); with a per-frame clock the dataplane raises them, which is
exact only when the stored value came from that clock, and not when the control plane wrote it (ses_touch and
ses_touch_exact; the EIM reuse of the ordered phase's nat_chunk_coop).

Every flow below starts from map updates (subscriber_nat, nat_sessions, nat_reverse, eim_table) that put its counters
a few frames short of a wrap of a low word, with high words at 0, 0x7FFFFFFF and 0xFFFFFFFF, or at 2^64 - 1, and its
stamps above, between, on and below the clocks of its frames.  Each flow has 1 to a few thousand frames scattered over
the whole batch, so that its atomics come from many warps and blocks at once.  Three batches alternate a per-frame clock
with one clock per batch; between them, half of the flows are put back on an edge by a control-plane update.  The
scripts run on the oracle and on the GPU (nat44_egress with EIM on and off, nat44_ingress, pipeline_up, pipeline_tc with
limited buckets, so that its hits go through the ordered phase), pageable, pinned and device-resident, and must agree
bit for bit.  A new-flow workload reuses pre-installed EIM mappings; one variant crosses the 16-bit epoch reset, one
puts the state in through bng_restore of a snapshot, and a seeded differential draws counters and stamps near the same
edges.

The tests without the gpu mark run every script on the oracle alone and check that each flow reaches the edge it was
built for (a high word moved, packets wrapped to 0 with bytes advanced by exactly the frame's length, last_seen ended
below the value written), and that the oracle's counters are the exact u64 sums."""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import pytest

import harness
from bng_b200 import layouts as L
from bng_b200 import synth as S

GW_MAC = 0x02FFFFFFFFFE
PUB0 = 0xCB007100       # subscriber s translates to PUB0 + s
DST0 = 0x08080800
NATF_EIM, NATF_HAIRPIN, NATF_ALG = 0x01, 0x04, 0x18
M32, M64 = (1 << 32) - 1, (1 << 64) - 1
HIS = (0, 0x7FFFFFFF, 0xFFFFFFFF)
N_SUBS = 48
T0 = 100 * 10**9
TICK = 1000             # per-frame clock: frame i of a batch runs at base + i * TICK
STAMPS = ("above", "between", "equal", "below")
EPOCH_PERIOD = 65535    # bng_prog_run: epoch = batch_seq % 65535 + 1, all cleared when it comes round to 1


def _need(kind):
    if kind == "none":
        pytest.fail("no oracle library present on this box")


# ---------------------------------------------------------------------------
# flows and the edges they start on
# ---------------------------------------------------------------------------
class Flow(NamedTuple):
    j: int
    sub: int
    sport: int
    dst: int
    proto: int
    nat_port: int
    nf: tuple       # frames per batch
    kind: str       # how its counters are put on an edge (seed_counters)
    k: int = 0      # packet low word at 0xFFFFFFFF - k
    delta: int = 0  # byte low word at 2^32 - (bytes of the batch) + delta
    ph: int = 0     # high words
    bh: int = 0
    stamp: str = "above"


def make_flow(j, nf, kind, **kw):
    return Flow(j, j % N_SUBS, 20000 + j, j % 7, 17 if j % 3 == 0 else 6, 1024 + j, tuple(nf), kind, **kw)


def seed_counters(f: Flow, lens):
    """(packets, bytes) that put flow f on its edge for a batch whose frames of f have lengths `lens`."""
    n, tot = len(lens), int(np.sum(lens, dtype=np.uint64))
    hi = lambda h, lo: (h << 32) | (lo & M32)
    if f.kind == "both":      # one frame: it wraps the packet word and, on its own, the byte word
        return hi(f.ph, M32), hi(f.bh, (1 << 32) - tot + f.delta)
    if f.kind == "spill":     # one frame: B + len = 2^32 - 1, so the spilled +1 is what wraps the byte word
        return hi(f.ph, M32), hi(f.bh, (1 << 32) - 1 - tot)
    if f.kind == "many":      # the packet word wraps k + 1 frames in, the byte word at the end (delta >= 0)
        return hi(f.ph, M32 - min(f.k, n - 1)), hi(f.bh, (1 << 32) - tot + f.delta)
    if f.kind == "race":      # the packet word wraps first; the byte word is one short of wrapping at the end, so a frame
        return hi(f.ph, M32), hi(f.bh, (1 << 32) - 1 - tot)  # that lands while the spill is in flight wraps it
    if f.kind == "pmax":      # packets = 2^64 - 1 (finding: the packets high half carried into the bytes high half)
        return M64, hi(f.bh, 0x12345678 + f.delta)
    if f.kind == "bmax":      # bytes one frame short of 2^64
        return hi(f.ph, 0x1000 + f.k), (M64 - tot + 1 + f.delta) & M64
    return hi(f.ph, 1000 + f.j), hi(f.bh, 5000 * f.j)  # "far": nowhere near a wrap


def edges_of(f: Flow, n):
    """What the flow must show after a batch with n of its frames that started from seed_counters."""
    if n == 0 or f.kind == "far":
        return set()
    if f.kind == "bmax":
        return {"by_hi"} if f.delta >= 0 else set()
    e = {"pk_hi"}  # every other kind wraps the packet low word
    if f.kind == "pmax" and n == 1:
        e.add("pk_zero")
    if f.kind in ("both", "many") and f.delta >= 0:
        e.add("by_hi")
    return e


def constructed_flows():
    fl, j = [], 0

    def add(nf, kind, **kw):
        nonlocal j
        fl.append(make_flow(j, nf, kind, stamp=STAMPS[j % 4] if min(x for x in nf if x) > 1 else ("above", "below")[j % 2],
                            **kw))
        j += 1
    for ph in HIS:
        for bh in HIS:
            add((1, 2, 1), "both", ph=ph, bh=bh)
            add((1, 1, 3), "both", ph=ph, bh=bh, delta=1)
            add((1, 3, 1), "spill", ph=ph, bh=bh)
    sizes = (2, 7, 40, 300, 2500)
    for i, (k, delta) in enumerate((k, d) for k in (0, 1, 5, 10**6) for d in (-1, 0, 1)):
        h = HIS[i % 3]
        add((sizes[i % 5], sizes[(i + 2) % 5], 5), "many", k=k, delta=delta, ph=h, bh=HIS[(i + 1) % 3])
    for i, h in enumerate(HIS):
        add((sizes[i + 1], 4, 2), "race", ph=h, bh=HIS[2 - i])
        add((1, 1, 1), "pmax", bh=h)
        add((1, 1, 1), "pmax", bh=h, delta=3)
        add((60, 2, 9), "pmax", bh=h, delta=7)
        add((1, 5, 1), "bmax", ph=h)
        add((30, 5, 1), "bmax", ph=h, delta=-1)
    for i in range(8):
        add((sizes[i % 5], 0 if i % 3 == 0 else 3, 2), "far", ph=HIS[i % 3])
    return fl


# ---------------------------------------------------------------------------
# state
# ---------------------------------------------------------------------------
def ses_key(f: Flow):
    k = np.zeros(1, L.nat_key)
    k["src_ip"], k["dst_ip"] = S.ip_bytes(S.sub_ip(f.sub)), S.ip_bytes(DST0 + f.dst)
    k["src_port"], k["dst_port"], k["protocol"] = S.port_bytes(f.sport), S.port_bytes(443), f.proto
    return k


def rev_key(f: Flow):
    k = np.zeros(1, L.nat_key)
    k["src_ip"], k["dst_ip"] = S.ip_bytes(DST0 + f.dst), S.ip_bytes(PUB0 + f.sub)
    k["src_port"], k["dst_port"], k["protocol"] = S.port_bytes(443), S.port_bytes(f.nat_port), f.proto
    return k


def ses_value(f: Flow, pk, by, last_seen):
    v = np.zeros(1, L.nat_session)
    v["nat_ip"], v["nat_port"] = S.ip_bytes(PUB0 + f.sub), S.port_bytes(f.nat_port)
    v["orig_port"], v["orig_ip"] = S.port_bytes(f.sport), S.ip_bytes(S.sub_ip(f.sub))
    v["dest_ip"], v["dest_port"] = S.ip_bytes(DST0 + f.dst), S.port_bytes(443)
    v["last_seen"], v["created"] = last_seen, T0 // 2
    v["packets_out"] = v["packets_in"] = pk
    v["bytes_out"] = v["bytes_in"] = by
    v["state"], v["protocol"] = 1, f.proto
    return v


def base_maps(sc, prog, eim):
    idx = np.arange(N_SUBS)
    v = np.zeros(N_SUBS, L.subscriber_nat)
    v["block"]["public_ip"] = S.ip_bytes(PUB0 + idx)
    v["block"]["port_start"], v["block"]["port_end"], v["block"]["next_port"] = 40000, 40999, 40000
    v["block"]["subscriber_id"] = idx + 1
    sc.update("subscriber_nat", S.ip_bytes(S.sub_ip(idx)), v)
    sc.update1("nat_config_map", np.uint32(0), S.nat_config(NATF_HAIRPIN | NATF_ALG | (NATF_EIM if eim else 0), 64))
    if prog.startswith("pipeline"):
        keys, b = S.bindings(N_SUBS)
        sc.update("subscriber_bindings", keys, b)
        cfg = np.zeros(1, L.antispoof_config)
        cfg["default_mode"] = 1
        sc.update1("antispoof_config", np.uint32(0), cfg)
        # limited buckets that pass everything: pipeline_tc runs every frame's NAT — hits too — in the ordered phase
        tb = np.zeros(N_SUBS, L.token_bucket)
        tb["rate_bps"], tb["burst_bytes"] = 10**12, 1 << 30
        tb["tokens"] = tb["burst_bytes"]
        sc.update("qos_ingress", S.ip_bytes(S.sub_ip(idx)), tb)
        sc.update("qos_egress", S.ip_bytes(S.sub_ip(idx)), tb)


# ---------------------------------------------------------------------------
# batches
# ---------------------------------------------------------------------------
def layout(r, flows, b):
    """Frame order of batch b: every flow's frames scattered over the whole batch.  (flow index per frame, lengths)"""
    owner = np.concatenate([np.full(f.nf[b], i, np.int64) for i, f in enumerate(flows)])
    owner = owner[r.permutation(len(owner))]
    proto = np.array([flows[i].proto for i in owner], np.uint32)
    lens = np.where(proto == 6, r.integers(54, 65, len(owner)), r.integers(42, 65, len(owner))).astype(np.uint32)
    return owner, lens


def frames(flows, owner, lens, ingress):
    sub = np.array([flows[i].sub for i in owner], np.int64)
    dst = np.array([DST0 + flows[i].dst for i in owner], np.uint32)
    proto = np.array([flows[i].proto for i in owner], np.uint32)
    sport = np.array([flows[i].sport for i in owner], np.uint32)
    ck = (0x1000 + np.arange(len(owner))).astype(np.uint32)
    if ingress:
        nport = np.array([flows[i].nat_port for i in owner], np.uint32)
        h = S.ipv4_headers(np.uint64(GW_MAC), S.sub_mac_key(sub), dst, (PUB0 + sub).astype(np.uint32), proto, 443, nport,
                           lens, l4_check=ck)
    else:
        h = S.ipv4_headers(S.sub_mac_key(sub), np.uint64(GW_MAC), S.sub_ip(sub), dst, proto, sport, 443, lens, l4_check=ck)
    return h.reshape(-1)


def stamp_value(pos, times, base):
    """A control-plane stamp at `pos` relative to the clocks `times` (sorted) of a flow's frames in the next batch."""
    if len(times) == 0:
        return base + 7
    t0, t1 = int(times[0]), int(times[-1])
    if pos == "above":
        return t1 + 10**12
    if pos == "between" and t1 > t0:
        return (t0 + t1) // 2 + TICK // 2  # (between two frames' clocks)
    if pos in ("between", "equal"):
        return int(times[len(times) // 2])
    return t0 - 1


class Built(NamedTuple):
    script: harness.Script
    setup: int          # steps before the first run (the map state a restore variant carries instead)
    flows: list
    seeds: list         # per batch: {flow index: (packets, bytes, last_seen)} written just before it
    owners: list        # per batch: (owner, lens)
    clocks: list
    lookups: list       # per batch: the result tag of each flow's nat_sessions lookup after it


def counters_script(name, flows, prog, eim, clocks, seed, wrap=False):
    """Setup, then one batch per clock kind ("frame" / "batch"), each followed by a lookup of every session.  Before
    every batch after the first, the flows with an odd index are put back on their edge (and their stamp) by a
    control-plane update.  wrap: idle batches before the last two, so that the batch-clock one is the last before the
    16-bit epoch reset and the per-frame one the batch that resets."""
    r = np.random.Generator(np.random.PCG64(seed))
    sc = harness.Script(name)
    base_maps(sc, prog, eim)
    ingress = prog == "nat44_ingress"
    lays = [layout(r, flows, b) for b in range(len(clocks))]
    bases = [T0 + b * 10**10 for b in range(len(clocks))]
    seeds, looks, batches = [], [], 0
    for b, clock in enumerate(clocks):
        owner, lens = lays[b]
        times = bases[b] + np.arange(len(owner), dtype=np.uint64) * TICK if clock == "frame" else None
        put = {}
        for i, f in enumerate(flows):
            if b and not f.j % 2:
                continue
            mine = owner == i
            pk, by = seed_counters(f, lens[mine])
            ls = stamp_value(f.stamp, times[mine], bases[b]) if clock == "frame" else bases[b] + 10**12
            put[i] = (pk, by, ls)
        if put:
            ks = np.concatenate([ses_key(flows[i]) for i in put])
            sc.update("nat_sessions", ks, np.concatenate([ses_value(flows[i], *v) for i, v in put.items()]))
            if b == 0:
                sc.update("nat_reverse", np.concatenate([rev_key(flows[i]) for i in put]), ks)
        if b == 0:
            setup = len(sc.steps)
        seeds.append(put)
        if wrap and b == len(clocks) - 2:  # idle batches up to the one before the reset
            arp = frames(flows, np.zeros(1, np.int64), np.full(1, 64, np.uint32), False)
            arp[12:14] = [0x08, 0x06]
            sc.repeat("antispoof_ingress", arp, np.full(1, 64, np.uint32), bases[b] - 1, EPOCH_PERIOD - 2 - batches)
            batches = EPOCH_PERIOD - 2
        sc.run(prog, frames(flows, owner, lens, ingress), lens, bases[b], stride=64, now_v=times)
        batches += 1
        tags = []
        for f in flows:  # every session after the batch (compared with the GPU's as well)
            tags.append(f"s{len(sc.steps):03d}")
            sc.lookup("nat_sessions", L.as_bytes(ses_key(f))[0])
        looks.append(tags)
    return Built(sc, setup, flows, seeds, lays, clocks, looks)


SCHEDULES = {"fbf": ("frame", "batch", "frame"), "bff": ("batch", "frame", "frame")}


def case_script(prog, eim, sched):
    return counters_script(f"counters/{prog}/{'eim' if eim else 'noeim'}/{sched}", constructed_flows(), prog, eim,
                           SCHEDULES[sched], seed=0xC0DE if sched == "fbf" else 0xC0DF)


def wrap_script(prog):
    # the batch-clock batch is the last one before the epoch reset, the per-frame one the batch that resets
    fl = [f._replace(nf=(f.nf[0], min(f.nf[1], 40), min(f.nf[2], 40))) for f in constructed_flows()]
    return counters_script(f"counters_wrap/{prog}", fl, prog, True, ("frame", "batch", "frame"), seed=0x3A9, wrap=True)


def random_flows(seed):
    r = np.random.Generator(np.random.PCG64(seed))
    fl = []
    for j in range(120):
        nf = tuple(int(r.choice([0, 1, 1, 2, 5, 30, 200, 800])) for _ in range(3))
        if nf[0] == 0:
            nf = (1,) + nf[1:]
        kind = str(r.choice(["both", "spill", "many", "many", "race", "pmax", "bmax", "far"]))
        fl.append(make_flow(j, nf, kind, k=int(r.choice([0, 1, 3, 64, 10**6])), delta=int(r.integers(-2, 3)),
                            ph=int(r.choice([0, 0x7FFFFFFF, M32, int(r.integers(0, 1 << 32))])),
                            bh=int(r.choice([0, 0x7FFFFFFF, M32, int(r.integers(0, 1 << 32))])),
                            stamp=str(r.choice(STAMPS))))
    return fl


def random_script(seed, prog):
    r = np.random.Generator(np.random.PCG64(seed + 1))
    clocks = tuple(str(c) for c in r.choice(["frame", "batch"], 3))
    return counters_script(f"counters_random/{seed:#x}/{prog}", random_flows(seed), prog, bool(seed & 1),
                           ("frame",) + clocks[1:], seed=seed)


# ---------------------------------------------------------------------------
# the EIM reuse workload: new flows from endpoints whose mapping exists (nat_chunk_coop, :482-487)
# ---------------------------------------------------------------------------
def eim_script(prog, seed=0xE1A):
    """Endpoints (subscriber, source port) with a pre-installed EIM mapping.  Every batch opens new flows from them to
    fresh destinations — several per endpoint and chunk, so lanes share a mapping — with a few repeated frames.  The
    mappings' last_used is written above, between, on and below the clocks of the frames that create flows; the batch
    kinds alternate, and the stamps are written again before the third batch.  Returns (script, what the third batch
    does: {"written": last_used written before it, "last": the clock of each mapping's last flow-creating frame,
    "created": flows created per mapping, "shared": 32-frame chunks of a subscriber's frames in which two or more
    flow-creating frames use one mapping})."""
    r = np.random.Generator(np.random.PCG64(seed))
    sc = harness.Script(f"eim_reuse/{prog}")
    base_maps(sc, prog, True)
    n_ep = 64
    ep_sub, ep_port = np.arange(n_ep) % N_SUBS, 30000 + np.arange(n_ep)
    ek = np.zeros(n_ep, L.eim_key)
    ek["internal_ip"] = S.ip_bytes(S.sub_ip(ep_sub))
    ek["internal_port"] = S.port_bytes(ep_port).view("<u2").reshape(-1)
    ek["protocol"] = 17
    clocks = ("frame", "batch", "frame")
    ndst = 0
    for b, clock in enumerate(clocks):
        ep = np.concatenate([np.full(int(r.choice([1, 2, 5, 33, 80])), e) for e in range(n_ep)])
        dst = np.arange(ndst, ndst + len(ep)) % 60000  # a new destination (a new flow) per frame ...
        ndst += len(ep)
        rep = r.integers(0, len(ep), len(ep) // 8)   # ... and some frames again
        ep, dst = np.concatenate([ep, ep[rep]]), np.concatenate([dst, dst[rep]])
        order = r.permutation(len(ep))
        ep, dst = ep[order], dst[order]
        n = len(ep)
        times = T0 + b * 10**10 + np.arange(n, dtype=np.uint64) * TICK if clock == "frame" else None
        if b != 1:
            m = np.zeros(n_ep, L.eim_mapping)
            m["external_ip"] = S.ip_bytes(PUB0 + ep_sub)
            m["external_port"] = 50000 + np.arange(n_ep)
            m["created"] = T0 // 2
            m["ref_count"] = 3
            _, first = np.unique(np.stack([ep, dst], 1), axis=0, return_index=True)
            for e in range(n_ep):  # the frames that create a flow of e read the mapping
                t = np.sort(times[first[ep[first] == e]])
                m["last_used"][e] = stamp_value(STAMPS[e % 4], t, T0)
            sc.update("eim_table", ek, m)
        lens = np.full(n, 60, np.uint32)
        h = S.ipv4_headers(S.sub_mac_key(ep_sub[ep]), np.uint64(GW_MAC), S.sub_ip(ep_sub[ep]),
                           (0x09000000 + dst).astype(np.uint32), 17, ep_port[ep], 53, lens, l4_check=0x4242)
        sc.run(prog, h.reshape(-1), lens, T0 + b * 10**10, stride=64, now_v=times)
    creating = np.zeros(n, bool)
    creating[first] = True
    shared = 0
    for s in range(N_SUBS):  # the ordered phase takes a subscriber's frames in index order, 32 at a time
        mine = np.flatnonzero(ep_sub[ep] == s)
        for c in range(0, len(mine), 32):
            ch = mine[c:c + 32]
            _, cnt = np.unique(ep[ch][creating[ch]], return_counts=True)
            shared += int((cnt >= 2).sum())
    info = {"written": m["last_used"].copy(), "shared": shared,
            "last": np.array([int(times[creating & (ep == e)].max()) for e in range(n_ep)], np.uint64),
            "created": np.array([int((creating & (ep == e)).sum()) for e in range(n_ep)])}
    return sc, info


# ---------------------------------------------------------------------------
# sessions the dataplane creates, then stamped under a per-frame clock after the epoch reset or a control-plane rewrite
# ---------------------------------------------------------------------------
def created_script(kind, prog, variant, seed=0xC4EA):
    """New flows created by `prog` in a fresh table (one clock per batch), then hit under a per-frame clock by `prog`
    and by nat44_ingress replies.  "wrap": the hits run in the batch that clears every epoch and the one after it.
    "update": before the hits, bng_map_update rewrites half of the sessions with the oracle's own values, but last_seen
    above, between, on and below the next frames' clocks.  A lookup of every session follows every batch.  The
    rewrite and the replies need the ports the dataplane hands out: they are read from the `kind` oracle's tables
    after the first batch.  Returns (script, {flow index: last_seen written}, index of the rewritten batch)."""
    r = np.random.Generator(np.random.PCG64(seed))
    fl = [make_flow(j, ((1, 3, 20, 150)[j % 4], (0, 2, 7, 40)[(j // 4) % 4], (1, 5)[j % 2], (2, 0, 6)[j % 3]), "far",
                    stamp=STAMPS[(j // 2) % 4])
          for j in range(160)]
    sc = harness.Script(f"created/{prog}/{variant}")
    base_maps(sc, prog, True)
    looks = []

    def run(p, b, clock, ingress):
        owner, lens = layout(r, fl, b)
        now = T0 + b * 10**10
        times = now + np.arange(len(owner), dtype=np.uint64) * TICK if clock == "frame" else None
        sc.run(p, frames(fl, owner, lens, ingress), lens, now, stride=64, now_v=times)
        for f in fl:
            sc.lookup("nat_sessions", L.as_bytes(ses_key(f))[0])
        return owner, times

    run(prog, 0, "batch", False)
    res = run_oracle(kind, sc)
    ses = final_sessions(res)
    vals = [ses[bytes(L.as_bytes(ses_key(f))[0])].copy() for f in fl]
    fl[:] = [f._replace(nat_port=int.from_bytes(bytes(v["nat_port"]), "big")) for f, v in zip(fl, vals)]
    written = {}
    if variant == "wrap":  # idle batches, so that the hits run in batches 65 535 (every epoch cleared) and 65 536
        arp = frames(fl, np.zeros(1, np.int64), np.full(1, 64, np.uint32), False)
        arp[12:14] = [0x08, 0x06]
        sc.repeat("antispoof_ingress", arp, np.full(1, 64, np.uint32), T0 + 1, EPOCH_PERIOD - 2)
        run(prog, 1, "frame", False)
        run("nat44_ingress", 2, "frame", True)
        return sc, written, None
    run(prog, 1, "frame", False)
    # the rewrite: the layout of batch 2 is drawn first, so that the stamps can be placed around its clocks
    state = r.bit_generator.state
    owner, _ = layout(r, fl, 2)
    r.bit_generator.state = state
    times = T0 + 2 * 10**10 + np.arange(len(owner), dtype=np.uint64) * TICK
    pick = [i for i in range(len(fl)) if i % 2]
    for i in pick:
        vals[i]["last_seen"] = written[i] = stamp_value(fl[i].stamp, times[owner == i], T0)
    sc.update("nat_sessions", np.concatenate([ses_key(fl[i]) for i in pick]), np.stack([vals[i] for i in pick]), 2)
    run(prog, 2, "frame", False)
    run("nat44_ingress", 3, "frame", True)
    return sc, written, 2


# ---------------------------------------------------------------------------
# reading the results
# ---------------------------------------------------------------------------
def final_sessions(res):
    """{session key bytes: nat_session record}"""
    k, v = res["tk_nat_sessions"], res["tv_nat_sessions"].view(L.nat_session).reshape(-1)
    return {bytes(kk): vv for kk, vv in zip(k, v)}


def check_edges(bt: Built, res, ingress):
    """On the oracle, after every batch: each flow put on an edge for it reached that edge, and every flow's counters
    are the exact u64 sums of what was written and the frames since.  Returns how often each edge was reached."""
    pk_f, by_f = ("packets_in", "bytes_in") if ingress else ("packets_out", "bytes_out")
    reached = dict.fromkeys(("pk_hi", "by_hi", "pk_zero", "ls_below"), 0)
    prev = {}
    for b, tags in enumerate(bt.lookups):
        owner, lens = bt.owners[b]
        for i, f in enumerate(bt.flows):
            s = res[tags[i] + "_val"].view(L.nat_session)[0]
            mine = lens[owner == i]
            n, tot = len(mine), int(np.sum(mine, dtype=np.uint64))
            pk0, by0, ls0 = bt.seeds[b][i] if i in bt.seeds[b] else prev[i]
            what = f"batch {b}, flow {f.j} ({f.kind}, k {f.k}, delta {f.delta}, hi {f.ph:#x}/{f.bh:#x}, {n} frames)"
            pk, by = int(s[pk_f]), int(s[by_f])
            assert (pk, by) == ((pk0 + n) & M64, (by0 + tot) & M64), f"{what}: the oracle's counters are not the u64 sums"
            prev[i] = (pk, by, int(s["last_seen"]))
            if i not in bt.seeds[b]:
                continue
            got = set()
            if pk >> 32 != pk0 >> 32:
                got.add("pk_hi")
            if by >> 32 != by0 >> 32:
                got.add("by_hi")
            if pk0 == M64 and n == 1 and pk == 0 and by == (by0 + tot) & M64:
                got.add("pk_zero")
            if int(s["last_seen"]) < ls0:
                got.add("ls_below")
            want = edges_of(f, n)
            if bt.clocks[b] == "frame" and f.stamp == "above" and n:
                want.add("ls_below")
            assert want <= got, f"{what}: built for {sorted(want)}, reached {sorted(got)}"
            for e in got:
                reached[e] += 1
    return reached


# ---------------------------------------------------------------------------
# GPU runs
# ---------------------------------------------------------------------------
GPU_OPTS = dict(max_subscribers=1 << 10, max_nat_sessions=1 << 14, max_eim_mappings=1 << 14, max_batch=1 << 15,
                event_capacity=1 << 16)


def run_oracle(kind, sc):
    be = harness.OracleBackend(kind)
    try:
        return harness.run_script(be, sc)
    finally:
        be.close()


class _DevWords:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}


def stats_vector(dp):
    """The dataplane's statistics vector (bng_stats_device_ptr), read from the device."""
    import torch
    dp.sync()
    ptr, n = dp.stats_device_ptr()
    return torch.as_tensor(_DevWords(ptr, n), device="cuda").cpu().numpy().copy()


ST_NAT_COOP = 37  # bng_b200/csrc/common.cuh: new flows committed by the ordered phase's cooperative chunks


def run_gpu(sc, feed, coop=False):
    """The results of a script on a fresh dataplane; coop: also how many new flows took the cooperative path."""
    be = harness.GpuBackend(pinned=feed, **GPU_OPTS)
    try:
        c0 = stats_vector(be.dp) if coop else None
        res = harness.run_script(be, sc)
        if coop:
            return res, int(stats_vector(be.dp)[ST_NAT_COOP] - c0[ST_NAT_COOP])
        return res
    finally:
        be.close()


def split(bt: Built):
    """(setup, runs): the script's map state and its batches as two scripts."""
    a, b = harness.Script(bt.script.name + "/setup"), harness.Script(bt.script.name)
    a.steps, b.steps = bt.script.steps[:bt.setup], bt.script.steps[bt.setup:]
    return a, b


CONFIGS = [("nat44_egress", False), ("nat44_egress", True), ("nat44_ingress", False), ("pipeline_up", True),
           ("pipeline_tc", True)]
CONFIG_IDS = ["egress_noeim", "egress_eim", "ingress", "pipeline_up", "pipeline_tc"]
FEEDS = [False, True, "device"]
FEED_IDS = ["pageable", "pinned", "device"]


# ---------------------------------------------------------------------------
# CPU: the oracle reaches every edge
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("sched", list(SCHEDULES))
@pytest.mark.parametrize("prog", ["nat44_egress", "nat44_ingress", "pipeline_tc"])
def test_cpu_cases_reach_their_edges(ora_kind, prog, sched):
    _need(ora_kind)
    bt = case_script(prog, prog != "nat44_ingress", sched)
    reached = check_edges(bt, run_oracle(ora_kind, bt.script), prog == "nat44_ingress")
    assert reached["pk_hi"] >= 30 and reached["by_hi"] >= 20 and reached["pk_zero"] >= 3 and reached["ls_below"] >= 5, \
        reached


def test_cpu_constructed_flows_cover_the_edges():
    fl = constructed_flows()
    kinds = {f.kind for f in fl}
    assert {"both", "spill", "many", "race", "pmax", "bmax", "far"} <= kinds
    assert {(f.ph, f.bh) for f in fl if f.kind == "both"} == {(p, b) for p in HIS for b in HIS}
    assert {f.delta for f in fl if f.kind == "many"} == {-1, 0, 1} and max(max(f.nf) for f in fl) >= 2000
    assert {f.stamp for f in fl} == set(STAMPS)
    assert sum(f.nf[0] for f in fl) <= GPU_OPTS["max_batch"]


def test_cpu_epoch_wrap_script_straddles_the_reset(ora_kind):
    _need(ora_kind)
    bt = wrap_script("nat44_egress")
    runs = [st for st in bt.script.steps if st[0] in ("run", "repeat")]
    assert sum(st[6] if st[0] == "repeat" else 1 for st in runs) == EPOCH_PERIOD
    assert runs[-2][0] == "run" and runs[-2][8] is None and runs[-1][8] is not None  # batch clock, then per-frame
    check_edges(bt, run_oracle(ora_kind, bt.script), False)


@pytest.mark.parametrize("seed", [0x5EED1, 0x5EED2])
def test_cpu_random_scripts_reach_the_edges(ora_kind, seed):
    _need(ora_kind)
    bt = random_script(seed, "nat44_egress")
    reached = check_edges(bt, run_oracle(ora_kind, bt.script), False)
    assert reached["pk_hi"] >= 10 and reached["by_hi"] >= 5 and reached["ls_below"] >= 3, reached


def test_cpu_eim_reuse_stamps_land_below(ora_kind):
    """On the oracle, after the third batch (per-frame clock): every mapping's last_used is the clock of the last frame
    that created a flow from it — so the ones written above their frames' clocks ended below the value written — and
    its ref_count counts those flows.  Many 32-frame chunks of the ordered phase have several lanes on one mapping."""
    _need(ora_kind)
    sc, info = eim_script("nat44_egress")
    res = run_oracle(ora_kind, sc)
    k = res["tk_eim_table"].view(L.eim_key).reshape(-1)
    m = res["tv_eim_table"].view(L.eim_mapping).reshape(-1)
    e = np.array([int.from_bytes(bytes(x["internal_port"].reshape(1).view(np.uint8)), "big") for x in k]) - 30000
    assert sorted(e.tolist()) == list(range(64))
    assert np.array_equal(m["last_used"], info["last"][e]), "last_used is not the last creating frame's clock"
    assert np.array_equal(m["ref_count"], 3 + info["created"][e])
    above = np.array([STAMPS[x % 4] == "above" for x in e])
    assert above.sum() == 16 and (m["last_used"][above] < info["written"][e][above]).all()
    assert info["shared"] >= 40, info["shared"]


@pytest.mark.parametrize("prog", ["nat44_egress", "pipeline_tc"])
def test_cpu_created_flows_rewritten_reach_their_edge(ora_kind, prog):
    """On the oracle: after the rewrite and the per-frame batch, every rewritten session that batch hit ended at the
    clock of its last frame, below the value written where that was above them."""
    _need(ora_kind)
    sc, written, b = created_script(ora_kind, prog, "update")
    res = run_oracle(ora_kind, sc)
    runs = [i for i, st in enumerate(sc.steps) if st[0] == "run"]
    n_fl = 160
    lk = runs[b] + 1  # the lookups after the rewritten batch
    below = 0
    for i, ls in written.items():
        v = res[f"s{lk + i:03d}_val"].view(L.nat_session)[0]
        if STAMPS[(i // 2) % 4] == "above":
            assert int(v["last_seen"]) < ls, f"flow {i}: last_seen {int(v['last_seen'])}, written {ls}"
            below += 1
    assert below == n_fl // 8


def test_cpu_created_wrap_script_hits_in_the_reset_batch(ora_kind):
    _need(ora_kind)
    sc, _, _ = created_script(ora_kind, "nat44_egress", "wrap")
    runs = [st for st in sc.steps if st[0] in ("run", "repeat")]
    seq = np.cumsum([st[6] if st[0] == "repeat" else 1 for st in runs])
    assert seq[-2] == EPOCH_PERIOD and runs[-2][8] is not None and runs[-1][8] is not None  # per-frame clocks


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("sched", list(SCHEDULES))
@pytest.mark.parametrize("cfg", range(len(CONFIGS)), ids=CONFIG_IDS)
def test_counters_and_stamps_gpu(ora_kind, cfg, sched):
    _need(ora_kind)
    prog, eim = CONFIGS[cfg]
    bt = case_script(prog, eim, sched)
    ref = run_oracle(ora_kind, bt.script)
    for feed, fid in zip(FEEDS, FEED_IDS):
        harness.compare(ref, run_gpu(bt.script, feed), f"{bt.script.name}/{fid}")


@pytest.mark.gpu
@pytest.mark.parametrize("prog", ["nat44_egress", "pipeline_up", "pipeline_tc"])
def test_eim_reuse_gpu(ora_kind, prog):
    _need(ora_kind)
    sc, _ = eim_script(prog)
    ref = run_oracle(ora_kind, sc)
    for feed, fid in zip(FEEDS, FEED_IDS):
        got, coop = run_gpu(sc, feed, coop=True)
        harness.compare(ref, got, f"{sc.name}/{fid}")
        assert coop > 1000, f"{sc.name}/{fid}: only {coop} new flows took the cooperative path"


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["wrap", "update"])
@pytest.mark.parametrize("prog", ["nat44_egress", "pipeline_tc"])
def test_created_flows_gpu(ora_kind, prog, variant):
    """Sessions the dataplane created, stamped under a per-frame clock in the batch that clears the epochs, or after
    bng_map_update rewrote them."""
    _need(ora_kind)
    sc, _, _ = created_script(ora_kind, prog, variant)
    ref = run_oracle(ora_kind, sc)
    for feed in (["device"] if variant == "wrap" else [False, "device"]):
        harness.compare(ref, run_gpu(sc, feed), f"{sc.name}/{feed}")


@pytest.mark.gpu
@pytest.mark.parametrize("prog", ["nat44_egress", "nat44_ingress", "pipeline_tc"])
def test_epoch_wrap_gpu(ora_kind, prog):
    _need(ora_kind)
    bt = wrap_script(prog)
    harness.compare(run_oracle(ora_kind, bt.script), run_gpu(bt.script, "device"), bt.script.name)


@pytest.mark.gpu
@pytest.mark.parametrize("prog", ["nat44_egress", "nat44_ingress", "pipeline_tc"])
def test_restored_state_gpu(ora_kind, prog):
    """The same flows, with the GPU's map state put in by bng_restore of a snapshot taken on another dataplane."""
    _need(ora_kind)
    bt = case_script(prog, True, "fbf")
    setup, runs = split(bt)
    ora = harness.OracleBackend(ora_kind)
    try:
        for st in setup.steps:
            assert ora.update(st[1], st[2], st[3], st[4]) == 0
        ref = harness.run_script(ora, runs)
    finally:
        ora.close()
    src = harness.GpuBackend(**GPU_OPTS)
    try:
        for st in setup.steps:
            assert src.update(st[1], st[2], st[3], st[4]) == 0
        blob = src.dp.snapshot()
    finally:
        src.close()
    be = harness.GpuBackend(pinned="device", **GPU_OPTS)
    try:
        be.dp.restore(blob)
        got = harness.run_script(be, runs)
    finally:
        be.close()
    harness.compare(ref, got, f"{bt.script.name}/restored")


@pytest.mark.gpu
@pytest.mark.parametrize("prog", ["nat44_egress", "nat44_ingress", "pipeline_up", "pipeline_tc"])
@pytest.mark.parametrize("seed", [0x5EED1, 0x5EED2])
def test_random_gpu(ora_kind, seed, prog):
    _need(ora_kind)
    bt = random_script(seed, prog)
    harness.compare(run_oracle(ora_kind, bt.script), run_gpu(bt.script, "device" if seed & 1 else False), bt.script.name)
