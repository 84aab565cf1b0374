"""nat44_ingress against the oracle on crowded flow tables, shared flows and stale reverse entries.

k_nat_ingress (bng_b200/csrc/kernels.cu) reads only the home slot of nat_reverse and of nat_sessions and falls back to
tbl_find when that slot holds anything but the key or EMPTY; it reloads the session's epoch when the session was found
off its home slot; a CAS-guarded erase decides which frame of a stale reverse entry counts sessions_expired; the TCP
state moves through a CAS loop on the state word; frames with IPv4 options and (bng_nat_icmp_errors_enable) ICMP
errors leave the warp's fast path for their own lane.  Every one of these is observable, and all of it is part of
bit-exact parity with the reference (DESIGN.md §3).

The tables here are small (max_nat_sessions 256: 512 slots, about 45 % full at the peak, never at max_entries, so no
LRU victim is involved) and the keys are chosen with a restatement of the device hash (common.cuh: hash_word,
tbl_hash<2>):
  * groups of flows whose reverse keys share one home slot and whose session keys share another, the group's anchor
    created one egress batch before its followers, so that the followers are displaced for certain; some homes are
    the last slot, so that those chains wrap to slot 0;
  * anchors deleted through the map commands (the followers' home slots become tombstones), some re-created (their
    session key lands on its old tombstone, their reverse key, with a new port, elsewhere);
  * sessions deleted underneath their reverse entries (stale), reverse entries deleted underneath their sessions,
    tuples never mapped, and replies whose reverse key's first word is one of the reserved slot states.
Then four reply batches: every flow with TCP, UDP (checksum 0 and not) and ICMP echo replies; hundreds of frames of
a few TCP flows starting in states 0, 1, 2 and 3 (2 and 3 written by the control plane) with mixed SYN-ACK / ACK /
FIN / RST / no-flag frames; one stale tuple hit by every frame of a 1 100-frame batch; and warps that mix ihl 5, 6
and 15, frames too short for their header, ICMP errors quoting the same flows, and a second stale tuple hit from five
warps.  The batches run with one clock per batch and with a per-frame clock, and ICMP error translation off and on
(the oracle side of that rule is test_gpu_nat_icmp's restatement).

The restated hash is checked against the device through the nat_reverse LRU rule (DESIGN.md §4: at capacity, the
victim is the first live slot from the new key's home).  The tests without the gpu mark check the restatement against
a scalar one, that the intended collisions and wraps are among the keys built, and that the oracle does what each
batch was built for."""
from __future__ import annotations

import numpy as np
import pytest

import harness
from bng_b200 import layouts as L
from bng_b200 import synth as S
from test_gpu_nat_icmp import IcmpBackend, RuleOracle, error_frame

GW_MAC = 0x02FFFFFFFFFE
N_SUBS = 16
PUB0 = 0xCB007100      # subscriber s translates to PUB0 + s
PORT0 = 40000          # every subscriber's port block starts here (on its own public address)
CAP = 256              # max_nat_sessions: nat_sessions and nat_reverse have 2 x 256 slots
SLOTS = 512
T0 = 50 * 10**9
FAR = 1 << 60          # a control-plane last_seen above every clock of the test
STRIDE = 128
GPU_OPTS = dict(max_subscribers=64, max_nat_sessions=CAP, max_eim_mappings=CAP, max_batch=1 << 13,
                event_capacity=1 << 14)
FEEDS = [False, True, "device"]
FEED_IDS = ["pageable", "pinned", "device"]
K_BUSY = 0xFFFFFFFFFFFFFFFD
ACK, SYNACK, FIN, RST, NOFLAG = 0x10, 0x12, 0x11, 0x04, 0x00


def _need(kind):
    if kind == "none":
        pytest.fail("no oracle library present on this box")


# ---------------------------------------------------------------------------
# the device hash, restated (bng_b200/csrc/common.cuh: hash_word, tbl_hash<2>)
# ---------------------------------------------------------------------------
def hash_word(k, seed):
    k = np.asarray(k, np.uint64)
    h = ((k & np.uint64(0xFFFFFFFF)).astype(np.uint32) * np.uint32(0x9E3779B1)) \
        ^ ((k >> np.uint64(32)).astype(np.uint32) * np.uint32(0x85EBCA77)) ^ np.asarray(seed, np.uint32)
    h ^= h >> np.uint32(16)
    h *= np.uint32(0x7FEB352D)
    h ^= h >> np.uint32(15)
    return h


def tbl_hash2(words):
    """tbl_hash<2> of u64[n, 2] key words."""
    return hash_word(words[:, 1], hash_word(words[:, 0], np.uint32(0x2545F491)))


def key_words(keys):
    return np.ascontiguousarray(L.as_bytes(keys)).reshape(-1, 16).view("<u8")


def home(keys, slots=SLOTS):
    return (tbl_hash2(key_words(keys)) & np.uint32(slots - 1)).astype(np.int64)


def home_scalar(key: bytes, slots=SLOTS):
    """The same hash on Python integers, one key at a time."""
    h = 0x2545F491
    for j in range(2):
        k = int.from_bytes(key[8 * j:8 * j + 8], "little")
        h = ((k & 0xFFFFFFFF) * 0x9E3779B1 ^ (k >> 32) * 0x85EBCA77 ^ h) & 0xFFFFFFFF
        h ^= h >> 16
        h = (h * 0x7FEB352D) & 0xFFFFFFFF
        h ^= h >> 15
    return h & (slots - 1)


# ---------------------------------------------------------------------------
# flows
# ---------------------------------------------------------------------------
class Flows:
    """One record per flow incarnation (a re-created flow is a new record with a new public port)."""
    FIELDS = ("sub", "proto", "rip", "rport", "sport", "nport", "ck", "batch")

    def __init__(self):
        self.cols = {f: [] for f in self.FIELDS}
        self.next_port = np.full(N_SUBS, PORT0, np.int64)

    def __len__(self):
        return len(self.cols["sub"])

    def col(self, f, idx=None):
        a = np.array(self.cols[f], np.int64)
        return a if idx is None else a[np.asarray(idx, np.int64)]

    def add(self, sub, proto, rip, rport, sport, batch, ck=None):
        """A flow created by the egress batch `batch`; its public port is the subscriber's next one (nat_config has no
        EIM and no port parity, so nat44_egress hands out a block's ports in frame order)."""
        for f, v in zip(self.FIELDS, (sub, proto, rip, 0 if proto == 1 else rport, sport, int(self.next_port[sub]),
                                      (0x1234 + len(self) * 7) & 0xFFFF if ck is None else ck, batch)):
            self.cols[f].append(int(v))
        self.next_port[sub] += 1
        return len(self) - 1

    def recreate(self, i, batch):
        return self.add(*(self.cols[f][i] for f in ("sub", "proto", "rip", "rport", "sport")), batch, self.cols["ck"][i])

    def ses_keys(self, idx):
        idx = np.atleast_1d(idx)
        k = np.zeros(len(idx), L.nat_key)
        k["src_ip"], k["dst_ip"] = S.ip_bytes(S.sub_ip(self.col("sub", idx))), S.ip_bytes(self.col("rip", idx))
        k["src_port"], k["dst_port"] = S.port_bytes(self.col("sport", idx)), S.port_bytes(self.col("rport", idx))
        k["protocol"] = self.col("proto", idx)
        return k

    def rev_keys(self, idx):
        idx = np.atleast_1d(idx)
        k = np.zeros(len(idx), L.nat_key)
        k["src_ip"], k["dst_ip"] = S.ip_bytes(self.col("rip", idx)), S.ip_bytes(PUB0 + self.col("sub", idx))
        k["src_port"], k["dst_port"] = S.port_bytes(self.col("rport", idx)), S.port_bytes(self.col("nport", idx))
        k["protocol"] = self.col("proto", idx)
        return k

    def egress_frames(self, idx):
        idx = np.atleast_1d(idx)
        sub = self.col("sub", idx)
        return S.ipv4_headers(S.sub_mac_key(sub), np.uint64(GW_MAC), S.sub_ip(sub), self.col("rip", idx),
                              self.col("proto", idx), self.col("sport", idx), self.col("rport", idx), 64,
                              l4_check=self.col("ck", idx), tcp_flags=0x02)

    def snat_frames(self, idx):
        """What nat44_egress sent out for these flows (the packets an ICMP error quotes)."""
        idx = np.atleast_1d(idx)
        sub = self.col("sub", idx)
        return S.ipv4_headers(S.sub_mac_key(sub), np.uint64(GW_MAC), PUB0 + sub, self.col("rip", idx),
                              self.col("proto", idx), self.col("nport", idx), self.col("rport", idx), 64,
                              l4_check=self.col("ck", idx), tcp_flags=0x02)

    def replies(self, idx, flags=ACK, width=64):
        """Replies u8[n, width] to flows idx (repeats allowed); TCP flags per frame."""
        idx = np.atleast_1d(idx)
        sub, proto = self.col("sub", idx), self.col("proto", idx)
        icmp = proto == 1
        h = S.ipv4_headers(np.uint64(GW_MAC), S.sub_mac_key(sub), self.col("rip", idx), PUB0 + sub, proto,
                           np.where(icmp, self.col("nport", idx), self.col("rport", idx)), self.col("nport", idx), 64,
                           l4_check=self.col("ck", idx), tcp_flags=np.broadcast_to(np.asarray(flags, np.uint8), len(idx)))
        h[icmp, 34] = 0  # echo reply
        out = np.zeros((len(idx), width), np.uint8)
        out[:, :64] = h
        return out


def find_tuple(r, fl: Flows, sub, proto, hr, hs, taken):
    """(rip, rport, sport) for a new flow of `sub` (its public port is the next one) whose reverse key has home hr and
    whose session key has home hs (None: anywhere), both keys new."""
    n = 1 << 14
    nport = int(fl.next_port[sub])
    for _ in range(50):
        rip = (0x09000000 + r.integers(0, 1 << 22, n)).astype(np.int64)
        rport = np.zeros(n, np.int64) if proto == 1 else r.integers(1024, 60000, n)
        rk = np.zeros(n, L.nat_key)
        rk["src_ip"], rk["dst_ip"] = S.ip_bytes(rip), S.ip_bytes(PUB0 + sub)
        rk["src_port"], rk["dst_port"], rk["protocol"] = S.port_bytes(rport), S.port_bytes(nport), proto
        ok = np.ones(n, bool) if hr is None else home(rk) == hr
        for j in np.flatnonzero(ok)[:4]:
            sport = r.integers(1024, 60000, n)
            sk = np.zeros(n, L.nat_key)
            sk["src_ip"], sk["dst_ip"] = S.ip_bytes(S.sub_ip(sub)), S.ip_bytes(rip[j])
            sk["src_port"], sk["dst_port"], sk["protocol"] = S.port_bytes(sport), S.port_bytes(rport[j]), proto
            good = np.ones(n, bool) if hs is None else home(sk) == hs
            for m in np.flatnonzero(good):
                if bytes(L.as_bytes(sk[m:m + 1])[0]) not in taken and bytes(L.as_bytes(rk[j:j + 1])[0]) not in taken:
                    taken.add(bytes(L.as_bytes(sk[m:m + 1])[0]))
                    taken.add(bytes(L.as_bytes(rk[j:j + 1])[0]))
                    return int(rip[j]), int(rport[j]), int(sport[m])
    raise AssertionError("no tuple found")


# group g: an anchor (egress batch 0) and three followers (batch 1), reverse keys on home RHOME[g], session keys on
# SHOME[g].  Groups 0-7 lose their anchor (the followers' home slots become tombstones); 0-3 get it back in batch 2.
N_GROUPS = 12
RHOME = [SLOTS - 1, 40, SLOTS - 2, 120, 160, 200, 240, 280, 320, 360, 400, 440]
SHOME = [20, SLOTS - 1, 100, SLOTS - 2, 180, 220, 260, 300, 340, 380, 420, 460]
GPROTO = [17, 1, 6, 6, 6, 6, 17, 1, 17, 6, 1, 17]
N_FILL = 180


class World:
    """The flows of the crowded-table script and what was done to them."""

    def __init__(self, seed=0x1A6E55):
        r = np.random.Generator(np.random.PCG64(seed))
        self.r = r
        fl = self.fl = Flows()
        taken = set()
        self.anchor, self.followers = [], []
        for g in range(N_GROUPS):
            self.anchor.append(fl.add(g % N_SUBS, GPROTO[g], *find_tuple(r, fl, g % N_SUBS, GPROTO[g], RHOME[g], SHOME[g],
                                                                         taken), 0))
        for g in range(N_GROUPS):
            fs = []
            for m in range(3):
                s = (g + 5 * m + 1) % N_SUBS
                fs.append(fl.add(s, GPROTO[g], *find_tuple(r, fl, s, GPROTO[g], RHOME[g], SHOME[g], taken), 1,
                                 ck=0 if (GPROTO[g] == 17 and m == 1) else None))
            self.followers.append(fs)
        self.fill = []
        for j in range(N_FILL):
            s, p = int(r.integers(0, N_SUBS)), int((6, 17, 17, 1)[j % 4])
            self.fill.append(fl.add(s, p, *find_tuple(r, fl, s, p, None, None, taken), 1,
                                    ck=0 if j % 8 == 1 else None))
        # S1 (UDP) and S2 (TCP): stale under contention
        self.s1 = next(i for i in self.fill[40:] if fl.cols["proto"][i] == 17 and fl.cols["ck"][i])
        self.s2 = next(i for i in self.fill[40:] if fl.cols["proto"][i] == 6)
        self.del_both = [self.anchor[g] for g in range(8)] + self.fill[:20]
        self.stale = self.fill[20:32] + [self.followers[8][0], self.followers[9][0]]
        self.del_rev = self.fill[32:37]
        self.recreated = [fl.recreate(self.anchor[g], 2) for g in range(4)] + [fl.recreate(i, 2) for i in self.fill[:10]]
        # hundreds of frames of a few TCP flows: followers of groups 2-5 (anchors back home in 2-3, tombstones in 4-5)
        tcp_f = [i for g in (2, 3, 4, 5) for i in self.followers[g]]
        self.states = {i: st for i, st in zip(tcp_f[:8], (0, 1, 2, 3, 3, 2, 1, 0))}  # control-plane written
        self.fresh0 = tcp_f[8:]                                                       # as nat44_egress made them
        # more TCP flows written back to state 0, for warps that race an ACK against a FIN (tcp_modes: "race")
        self.states.update((i, 0) for i in [i for i in self.fill[60:] if fl.cols["proto"][i] == 6 and i != self.s2][:6])
        self.rewritten = [self.followers[g][m] for g in (8, 9, 10, 11) for m in (1, 2)]  # last_seen FAR, epoch 0
        gone = set(self.del_both) | set(self.stale) | {self.s1, self.s2}
        self.live = [i for i in range(len(fl)) if i not in gone and i not in self.del_rev]

    def tcp_modes(self):
        """The TCP flags of each R2 flow's frames: "race" one warp of 31 ACKs and one FIN or RST, all reading state 0
        and racing for the state word; "ack" no FIN or RST, "noflag" no flag at all, "mixed" a few FIN and RST among
        hundreds of frames."""
        m = {}
        for k, (i, st) in enumerate(self.states.items()):
            m[i] = "race" if st == 0 else ("ack" if k < 4 and st in (1, 2) else "mixed")
        m.update(zip(self.fresh0, ("race", "race", "ack", "noflag")))
        return m

    def tcp_end_state(self, i):
        mode, st = self.tcp_modes()[i], self.states.get(i, 0)
        return {"race": 3, "mixed": 3, "noflag": st, "ack": 1 if st == 0 else st}[mode]

    # ---- frames ----
    def ingress_run(self, sc, rows, lens, clock, base, stride):
        n = len(lens)
        now_v = (base + np.cumsum(self.r.integers(1, 3000, n))).astype(np.uint64) if clock == "frame" else None
        arena = np.zeros((n, stride), np.uint8)
        arena[:, :rows.shape[1]] = rows[:, :stride]
        sc.run("nat44_ingress", arena.reshape(-1), np.asarray(lens, np.uint32), base, stride=stride, now_v=now_v)
        return len(sc.steps) - 1


def ses_value(fl: Flows, i, state, last_seen):
    v = np.zeros(1, L.nat_session)
    v["nat_ip"], v["nat_port"] = S.ip_bytes(PUB0 + fl.cols["sub"][i]), S.port_bytes(fl.cols["nport"][i])
    v["orig_port"], v["orig_ip"] = S.port_bytes(fl.cols["sport"][i]), S.ip_bytes(S.sub_ip(fl.cols["sub"][i]))
    v["dest_ip"], v["dest_port"] = S.ip_bytes(fl.cols["rip"][i]), S.port_bytes(fl.cols["rport"][i])
    v["last_seen"], v["created"] = last_seen, T0
    v["packets_out"], v["packets_in"], v["bytes_out"], v["bytes_in"] = 3, 5, 300, 500 + i
    v["state"], v["protocol"] = state, fl.cols["proto"][i]
    return v


def reserved_replies():
    """Replies to 255.255.255.255 whose reverse key's first word is K_EMPTY, K_TOMB or K_BUSY (source 255.255.255.255,
    254.255.255.255, 253.255.255.255), and their byte-swapped neighbours (255.255.255.253 / 254), TCP, UDP and ICMP."""
    srcs = [0xFFFFFFFF, 0xFEFFFFFF, 0xFDFFFFFF, 0xFFFFFFFE, 0xFFFFFFFD]
    rows = []
    for s in srcs:
        for p in (6, 17, 1):
            h = S.ipv4_headers(np.uint64(GW_MAC), S.sub_mac_key(0), s, 0xFFFFFFFF, p, 0xFFFF, 0xFFFF, 64,
                               l4_check=0xFFFF)
            rows.append(h[0])
    return np.stack(rows)


def with_options(f, ihl):
    """Frame f (ihl 5) with ihl - 5 words of NOP options: its L4 header moves on."""
    g = np.zeros_like(f)
    extra = 4 * (ihl - 5)
    g[:34] = f[:34]
    g[34:34 + extra] = 1
    g[34 + extra:] = f[34:len(f) - extra]
    g[14] = 0x40 | ihl
    return g


def ingress_script(clock="batch", seed=0x1A6E55):
    """Setup, then the four reply batches.  Returns (script, world, {batch name: step index})."""
    w = World(seed)
    fl, r = w.fl, np.random.Generator(np.random.PCG64(seed + 1))
    sc = harness.Script(f"nat_ingress/{clock}")
    idx = np.arange(N_SUBS)
    v = np.zeros(N_SUBS, L.subscriber_nat)
    v["block"]["public_ip"] = S.ip_bytes(PUB0 + idx)
    v["block"]["port_start"], v["block"]["port_end"], v["block"]["next_port"] = PORT0, PORT0 + 999, PORT0
    v["block"]["subscriber_id"] = idx + 1
    sc.update("subscriber_nat", S.ip_bytes(S.sub_ip(idx)), v)
    sc.update1("nat_config_map", np.uint32(0), S.nat_config(0, 1000))
    steps = {}
    batch = fl.col("batch")
    for b in range(3):
        if b == 2:  # deletions through the map commands, then batch 2 re-creates some of them
            for i in w.del_both:
                sc.delete("nat_sessions", L.as_bytes(fl.ses_keys(i))[0]).delete("nat_reverse", L.as_bytes(fl.rev_keys(i))[0])
            for i in w.stale + [w.s1, w.s2]:
                sc.delete("nat_sessions", L.as_bytes(fl.ses_keys(i))[0])
            for i in w.del_rev:
                sc.delete("nat_reverse", L.as_bytes(fl.rev_keys(i))[0])
        mine = np.flatnonzero(batch == b)
        sc.run("nat44_egress", fl.egress_frames(mine).reshape(-1), np.full(len(mine), 64, np.uint32), T0 + b * 10**9,
               stride=64)
        steps[f"egress{b}"] = len(sc.steps) - 1

    # ---- R1: every flow, crowded tables (case 1), reserved patterns, never-mapped tuples ----
    every = [i for i in range(len(fl)) if i not in (w.s1, w.s2) and i not in w.fresh0]  # (R2 starts those in state 0)
    who = np.repeat(every, r.integers(1, 4, len(every)))
    flags = r.choice(np.array([ACK, SYNACK, NOFLAG, ACK | 0x08], np.uint8), len(who))
    rows = [fl.replies(who, flags)]
    stray = fl.replies(r.choice(every, 40))  # never mapped: another remote port / address
    stray[:20, 34] ^= 0x5A
    stray[20:, 28] ^= 0x77
    rows += [stray, reserved_replies()]
    rows = np.concatenate(rows)
    order = r.permutation(len(rows))
    steps["crowded"] = w.ingress_run(sc, rows[order], np.full(len(rows), 64), clock, T0 + 10 * 10**9, 64)

    # ---- control-plane writes: TCP states 0-3, and displaced sessions with last_seen above every clock ----
    for i, st in w.states.items():
        sc.update("nat_sessions", fl.ses_keys(i), ses_value(fl, i, st, FAR))
    for i in w.rewritten:
        sc.update("nat_sessions", fl.ses_keys(i), ses_value(fl, i, 1, FAR), 2)

    # ---- R2: hundreds of frames of a few TCP flows (case 3); their home slots' flows early in the batch ----
    lead = [w.anchor[g] for g in (8, 9, 10, 11)] + w.recreated[:4]
    who, fla, race = [], [], []
    for i, mode in w.tcp_modes().items():
        if mode == "race":
            race.append(i)
            continue
        n = int(r.integers(250, 350))
        f = r.choice(np.array([ACK, SYNACK, NOFLAG, FIN, RST], np.uint8), n, p=[0.4, 0.2, 0.3, 0.05, 0.05])
        if mode != "mixed":
            f = np.where((f == FIN) | (f == RST), ACK, f)
        if mode == "noflag":
            f[:] = NOFLAG
        who.append(np.full(n, i))
        fla.append(f)
    who, fla = np.concatenate(who), np.concatenate(fla)
    order = r.permutation(len(who))
    who, fla = who[order], fla[order]
    # the race warps open the batch (warp-aligned): the FIN / RST lane at 31, 0, 16, ...
    rw, rf = np.repeat(race, 32), np.full(32 * len(race), ACK, np.uint8)
    for k in range(len(race)):
        rf[32 * k + (31, 0, 16, 30, 1, 15)[k % 6]] = FIN if k % 2 else RST
    early = np.repeat(lead, 24)
    who = np.concatenate([rw, early, who, w.rewritten])
    fla = np.concatenate([rf, np.full(len(early), ACK, np.uint8), fla, np.full(len(w.rewritten), ACK, np.uint8)])
    steps["one_flow"] = w.ingress_run(sc, fl.replies(who, fla), np.where(fl.col("proto", who) == 6, 60, 64), clock,
                                      T0 + 20 * 10**9, 64)

    # ---- R3: one stale tuple hit by every frame of a batch (case 4) ----
    n3 = 1100
    steps["stale_all"] = w.ingress_run(sc, fl.replies(np.full(n3, w.s1)), np.full(n3, 64), clock, T0 + 30 * 10**9, 64)

    # ---- R4: mixed warps (case 5) and a second stale tuple hit from five warps ----
    mixed = w.live[::3] + w.followers[4] + w.followers[6] + w.stale[:4]
    rows, lens = [], []
    for i in mixed:
        base = fl.replies(np.array([i, i, i]), np.array([ACK, SYNACK, FIN], np.uint8), width=STRIDE)
        p = fl.cols["proto"][i]
        need = 20 if p == 6 else 8
        rows += [base[0], with_options(base[1], 6), with_options(base[2], 15)]
        lens += [64, 68, 104]
        cut = with_options(base[0], (5, 6, 15)[i % 3])
        rows.append(cut)
        lens.append(14 + 4 * (5, 6, 15)[i % 3] + need - 1)  # one byte short of its L4 header
        e, el = error_frame(fl.snat_frames(i)[0], (28, 48)[i % 2], (3, 11, 12)[i % 3], 1)
        rows.append(e)
        lens.append(el)
    rows.append(fl.replies(np.array([w.live[0]]), width=STRIDE)[0])
    lens.append(33)  # too short for an IPv4 header
    rows, lens = np.stack(rows), np.array(lens)
    order = r.permutation(len(rows))
    rows, lens = rows[order], lens[order]
    s2 = fl.replies(np.full(5, w.s2), np.array([ACK, FIN, RST, NOFLAG, SYNACK], np.uint8), width=STRIDE)
    for k, at in enumerate((3, 200, 450, 777, 1100)):
        at = min(at, len(rows))
        rows = np.insert(rows, at, s2[k], axis=0)
        lens = np.insert(lens, at, 64)
    steps["mixed"] = w.ingress_run(sc, rows, lens, clock, T0 + 40 * 10**9, STRIDE)
    return sc, w, steps


# ---------------------------------------------------------------------------
# running
# ---------------------------------------------------------------------------
def run_oracle(kind, sc, icmp=False):
    be = RuleOracle(kind, on=icmp)
    try:
        return harness.run_script(be, sc)
    finally:
        be.close()


def run_gpu(sc, feed, icmp=False):
    be = IcmpBackend(pinned=feed, on=icmp, **GPU_OPTS)
    try:
        return harness.run_script(be, sc)
    finally:
        be.close()


def upto(sc, step):
    out = harness.Script(sc.name)
    out.steps = sc.steps[:step + 1]
    return out


def nat_stats(res):
    return dict(zip(L.nat_stats.names, res["st_nat_stats_map"][:len(L.nat_stats.names)].tolist()))


def rows_of(res, m):
    return {bytes(k) for k in res["tk_" + m]}


# ---------------------------------------------------------------------------
# CPU: the restatement, the keys built, and what the oracle does with them
# ---------------------------------------------------------------------------
def test_hash_restatement_self_consistent():
    r = np.random.Generator(np.random.PCG64(7))
    keys = r.integers(0, 256, (500, 16), dtype=np.uint8)
    keys[:3, :8] = 0xFF  # word 0 near the reserved patterns (the hash does not care)
    want = [home_scalar(bytes(k)) for k in keys]
    assert home(keys).tolist() == want
    assert home(keys, 64).tolist() == [home_scalar(bytes(k), 64) for k in keys]
    # every slot is somebody's home: the hash spreads 16-byte keys over a 512-slot table
    assert len(set(home(r.integers(0, 256, (20000, 16), dtype=np.uint8)).tolist())) == SLOTS


def test_keys_collide_and_wrap():
    """The groups share their home slots (reverse and session) as built, some of them the last slot, the anchors are
    alone on their homes, and every table stays below max_entries at about 40-45 % occupancy."""
    w = World()
    fl = w.fl
    rk, sk = fl.rev_keys(np.arange(len(fl))), fl.ses_keys(np.arange(len(fl)))
    rh, sh = home(rk), home(sk)
    for g in range(N_GROUPS):
        grp = [w.anchor[g]] + w.followers[g]
        assert set(rh[grp].tolist()) == {RHOME[g]} and set(sh[grp].tolist()) == {SHOME[g]}, g
    assert {SLOTS - 1, SLOTS - 2} <= set(RHOME) and {SLOTS - 1, SLOTS - 2} <= set(SHOME)
    # three live followers on the last slot and three on the one before, in either table: linear probing puts at least
    # two of each three at slot 0 or beyond
    for h in (SLOTS - 1, SLOTS - 2):
        assert sum(rh[i] == h for i in w.live) >= 3 and sum(sh[i] == h for i in w.live) >= 3, h
    assert len({rh[w.anchor[g]] for g in range(N_GROUPS)}) == N_GROUPS
    assert len({sh[w.anchor[g]] for g in range(N_GROUPS)}) == N_GROUPS
    assert sorted(i for i in range(len(fl)) if fl.cols["batch"][i] == 0) == w.anchor  # alone in the first batch
    # all keys distinct, reserved patterns never stored
    assert len({bytes(x) for x in L.as_bytes(sk)}) == len(fl) - len(w.recreated)  # re-created flows keep their key
    assert len({bytes(x) for x in L.as_bytes(rk)}) == len(fl)
    assert (key_words(rk)[:, 0] < K_BUSY).all() and (key_words(sk)[:, 0] < K_BUSY).all()
    peak = len(fl) - len(w.recreated)
    assert 0.40 * SLOTS <= peak < CAP - 16, peak
    # displaced sessions that the per-frame batch reaches with epoch 0 and a home slot another flow stamped
    assert all(sh[i] == SHOME[g] for g in (8, 9, 10, 11) for i in w.followers[g])
    # tombstones on the followers' home slots (anchors of groups 4-7 deleted and not re-created)
    assert all(w.anchor[g] in w.del_both for g in range(8))


@pytest.mark.parametrize("clock", ["batch", "frame"])
def test_oracle_does_what_the_batches_are_for(ora_kind, clock):
    _need(ora_kind)
    sc, w, steps = ingress_script(clock)
    fl = w.fl
    res = run_oracle(ora_kind, sc)
    # the public ports were predicted right: every live flow's reverse key is in the oracle's nat_reverse after the
    # egress batches (those R1 did not erase), and every egress frame created a session
    after = run_oracle(ora_kind, upto(sc, steps["egress2"]))
    rev = rows_of(after, "nat_reverse")
    for i in w.live + w.stale + [w.s1, w.s2]:
        assert bytes(L.as_bytes(fl.rev_keys(i))[0]) in rev, i
    assert nat_stats(after)["sessions_created"] == len(fl)
    assert len(after["tk_nat_reverse"]) == len(w.live) + len(w.stale) + 2
    # R1: the stale tuples expire once each, nothing is dropped
    part = {k: run_oracle(ora_kind, upto(sc, steps[k])) for k in ("egress2", "crowded", "one_flow", "stale_all")}
    s = [nat_stats(x) for x in part.values()] + [nat_stats(res)]
    assert s[1]["sessions_expired"] - s[0]["sessions_expired"] == len(w.stale)
    assert s[1]["packets_dnat"] - s[0]["packets_dnat"] > 300
    # R3: one stale tuple, 1 100 frames: one expiry, the rest passed, the entry gone
    assert s[3]["sessions_expired"] - s[2]["sessions_expired"] == 1
    assert s[3]["packets_passed"] - s[2]["packets_passed"] == 1099
    assert s[3]["packets_dnat"] == s[2]["packets_dnat"]
    # R4: the second stale tuple expires once, from five warps
    assert s[4]["sessions_expired"] - s[3]["sessions_expired"] == 1
    final = rows_of(res, "nat_reverse")
    for i in (w.s1, w.s2, *w.stale):
        assert bytes(L.as_bytes(fl.rev_keys(i))[0]) not in final
    # R2: the TCP flows end in every state; state-0 flows whose ACKs raced a FIN or RST end closing
    r2 = part["one_flow"]
    ses = {bytes(k): v for k, v in zip(r2["tk_nat_sessions"], r2["tv_nat_sessions"].view(L.nat_session).reshape(-1))}
    st = {i: int(ses[bytes(L.as_bytes(fl.ses_keys(i))[0])]["state"]) for i in list(w.states) + w.fresh0}
    assert st == {i: w.tcp_end_state(i) for i in st} and set(st.values()) == {0, 1, 2, 3}
    # the sessions written with last_seen above every clock ended at the clock of their last frame
    for i in w.rewritten + list(w.states):
        assert int(ses[bytes(L.as_bytes(fl.ses_keys(i))[0])]["last_seen"]) < FAR, i


def test_oracles_agree(oracle_kinds):
    if len(oracle_kinds) < 2:
        pytest.skip("the reference oracle is not built")
    for clock in ("batch", "frame"):
        sc, _, _ = ingress_script(clock)
        for icmp in (False, True):
            harness.compare(run_oracle("reference", sc, icmp), run_oracle("port", sc, icmp), f"{sc.name}/icmp={icmp}")


# ---------------------------------------------------------------------------
# the nat_reverse LRU rule on a 64-slot table, modelled with the restated hash
# ---------------------------------------------------------------------------
LRU_SLOTS, LRU_MAX = 64, 32
EMPTY, TOMB = None, "tomb"


def lru_keys(seed=0x64):
    """32 keys with the even homes 0, 2, .., 62, and new keys whose victims the model below predicts: homes 1 (victim
    at 2), 63 (its window wraps: victim at 0), 10 (a live home: its own key goes), 2 (a tombstone home: the next live
    key) and 40."""
    r = np.random.Generator(np.random.PCG64(seed))
    k = r.integers(0, 256, (1 << 14, 16), dtype=np.uint8)
    k[:, 7] &= 0x7F
    h = home(k, LRU_SLOTS)
    base = np.stack([k[np.flatnonzero(h == s)[0]] for s in range(0, LRU_SLOTS, 2)])
    new = np.stack([k[np.flatnonzero(h == s)[1]] for s in (1, 63, 10, 2, 40)])
    return base, new


def lru_model(base, new):
    """The table after each insert of `new`: tbl_find_or_claim (first tombstone on the path, else the EMPTY slot that
    ends it) with tbl_evict_near's LRU_ANY victim (the first live slot of the 16 from the new key's home)."""
    t = [EMPTY] * LRU_SLOTS
    for k in base:
        t[home_scalar(bytes(k), LRU_SLOTS)] = bytes(k)
    out, victims = [], []
    for k in new:
        hm = home_scalar(bytes(k), LRU_SLOTS)
        i, tomb = hm, None
        while t[i] is not EMPTY:
            if t[i] is TOMB and tomb is None:
                tomb = i
            i = (i + 1) % LRU_SLOTS
        target = tomb if tomb is not None else i
        v = next((hm + j) % LRU_SLOTS for j in range(16) if t[(hm + j) % LRU_SLOTS] not in (EMPTY, TOMB))
        victims.append(v)
        t[v] = TOMB
        t[target] = bytes(k)
        out.append({x for x in t if x not in (EMPTY, TOMB)})
    return out, victims


def test_lru_model_covers_the_edges():
    base, new = lru_keys()
    assert home(base, LRU_SLOTS).tolist() == list(range(0, LRU_SLOTS, 2))
    _, victims = lru_model(base, new)
    assert victims == [2, 0, 10, 4, 40], victims  # 0: the window of home 63 wrapped


@pytest.mark.gpu
def test_hash_matches_device_lru_victims():
    """At capacity, each insert into nat_reverse evicts the entry the restated hash predicts."""
    base, new = lru_keys()
    want, _ = lru_model(base, new)
    be = harness.GpuBackend(max_subscribers=64, max_nat_sessions=LRU_MAX, max_eim_mappings=64, max_batch=64,
                            event_capacity=1024)
    try:
        assert be.dp.map_info("nat_reverse")["max_entries"] == LRU_MAX
        vals = np.repeat(np.arange(len(base), dtype=np.uint8)[:, None], 16, axis=1)
        assert be.update("nat_reverse", base, vals, 0) == 0
        before = {bytes(x) for x in base}
        assert {bytes(x) for x in be.dump("nat_reverse")[0]} == before
        for j, k in enumerate(new):
            assert be.dp.update("nat_reverse", k, np.full(16, j, np.uint8)) == 0
            got = {bytes(x) for x in be.dump("nat_reverse")[0]}
            gone = sorted(home_scalar(x, LRU_SLOTS) for x in before - got)
            assert got == want[j], f"insert {j} (home {home_scalar(bytes(k), LRU_SLOTS)}): evicted the key of home {gone}"
            before = got
    finally:
        be.close()


# ---------------------------------------------------------------------------
# GPU: parity
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("icmp", [False, True], ids=["icmp_off", "icmp_on"])
@pytest.mark.parametrize("clock", ["batch", "frame"])
def test_ingress_gpu(ora_kind, clock, icmp):
    _need(ora_kind)
    sc, _, _ = ingress_script(clock)
    ref = run_oracle(ora_kind, sc, icmp)
    for feed, fid in zip(FEEDS, FEED_IDS):
        harness.compare(ref, run_gpu(sc, feed, icmp), f"{sc.name}/icmp={icmp}/{fid}")
