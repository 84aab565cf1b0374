"""The NAT flow tables at capacity, bit for bit against the oracle.

nat_sessions, nat_reverse and eim_table are BPF_MAP_TYPE_LRU_HASH (bpf/nat44.c:218-244): a BNG that has run for a
while keeps them full and evicts on every new flow.  The CPU oracle does not model LRU, and which entry gives way is
not part of parity (DESIGN.md §8).  What is: a correct dataplane equals the sequential reference with an LRU that
removes SOME entries at SOME moments.  `Replay` reproduces such a run from what the device shows, deleting each
victim on the oracle as late as the observations allow:

  * a SESSION_CREATE record of frame i for tuple T: before frame i, the oracle's session T (if it still has one) was
    evicted, and so was the EIM mapping of T's endpoint if its external port differs from the record's;
  * after the batch, a key the oracle holds and the device does not was evicted and not recreated.

Everything else — verdicts, frames, every counter, the event records, every table — must then be equal, and every
deletion must have been needed: a table the replay deleted from in a batch overflowed in it.  A slot used after it was
evicted and reclaimed (another flow's translation, a packet or an EIM reference counted on somebody else's entry)
leaves a state no such run explains.

The replay is exact while (1) port blocks do not wrap, so a recreated EIM mapping always gets a new port, and (2) no
source port, loaded little-endian, falls inside a port block (allocate_port_from_block probes eim_table with the
host-order candidate, bpf/nat44.c:450-455, so the port chosen would depend on when an eviction happened).  The
workloads below keep both.  The tests without the gpu mark check the checker on an oracle-backed fake dataplane."""
import os
import shutil
import time

import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import layouts as L
from bng_b200 import synth as S
from test_gpu_natuse import check_census
from test_gpu_sweep import MAPS as SWEEP_MAPS
from test_gpu_sweep import sweep_spec

LRU = ("nat_sessions", "nat_reverse", "eim_table")
SES_CAP, EIM_CAP = 2048, 1024
N_SUBS = 300            # subscribers with a 512-port block, 8 to a public address: ports 1024..5119
FAT = N_SUBS            # one more with 8192 ports on an address of its own: ports 1024..9215
FAT_IP = 0xCB00F000
DPORTS = np.array([443, 80, 53], np.uint32)  # no ALG port
NS = 10**9


@pytest.fixture(scope="module")
def lru_oracle():
    """One oracle: the reference's own sources when built, else the port (each test here takes seconds of oracle time)."""
    from oracle import pyoracle
    kinds = [k for k in ("reference", "port") if pyoracle.available(k)]
    if not kinds:
        pytest.fail("no oracle library present on this box")
    return kinds[0]


# ---------------------------------------------------------------------------
# traffic: flow u of subscriber s.  Three flows share an endpoint (source address, port, protocol), so EIM hits happen;
# every source port has a low byte >= 0x24, so loaded little-endian it is >= 0x2400 = 9216, above every block.
# ---------------------------------------------------------------------------
def flow_frames(sub, u) -> np.ndarray:
    sub, u = np.asarray(sub, np.int64), np.asarray(u, np.int64)
    v, k = u // 3, u % 3
    sport = ((1 + (v // 220) % 250) << 8) | (0x24 + v % 220)
    proto = np.where(v % 3 == 0, 17, 6).astype(np.uint32)
    lens = np.full(len(sub), 64, np.uint32)
    return S.ipv4_headers(S.sub_mac_key(sub), np.uint64(scenarios.GW_MAC), S.sub_ip(sub), (0x08080800 + k).astype(np.uint32),
                          proto, sport.astype(np.uint32), DPORTS[k], lens, l4_check=(0x1000 + (u & 0xFFF)).astype(np.uint32))


def maps_script(flags, prog) -> harness.Script:
    sc = harness.Script("lru_maps")
    scenarios.nat_maps(sc, N_SUBS, 512, flags)
    fk, fv, _ = S.nat_blocks(1, first_public_ip=FAT_IP, ports_per_sub=8192)
    fv["block"]["subscriber_id"] = FAT + 1
    sc.update("subscriber_nat", S.ip_bytes(S.sub_ip(np.array([FAT]))), fv)
    if prog.startswith("pipeline"):
        keys, v = S.bindings(N_SUBS + 1)
        sc.update("subscriber_bindings", keys, v)
        cfg = np.zeros(1, L.antispoof_config)
        cfg["default_mode"] = 1
        sc.update1("antispoof_config", np.uint32(0), cfg)
        # half the subscribers have a bucket: pipeline_tc runs their frames' NAT after it, in the ordered phase
        limited = np.arange(0, N_SUBS + 1, 2)
        tb = np.zeros(len(limited), L.token_bucket)
        tb["rate_bps"], tb["burst_bytes"] = 10**12, 1 << 30
        tb["tokens"] = tb["burst_bytes"]
        sc.update("qos_ingress", S.ip_bytes(S.sub_ip(limited)), tb)
        sc.update("qos_egress", S.ip_bytes(S.sub_ip(limited)), tb)
    return sc


class Traffic:
    """New flows and hits on older ones, with a strictly increasing clock across the whole test."""

    def __init__(self, seed):
        self.r = np.random.Generator(np.random.PCG64(seed))
        self.next_u = np.zeros(N_SUBS + 1, np.int64)
        self.batches = []  # (sub, u) of every batch's new flows
        self.t = 50 * NS

    def new(self, sub):
        sub = np.asarray(sub, np.int64)
        u = np.zeros(len(sub), np.int64)
        for i, s in enumerate(sub):
            u[i] = self.next_u[s]
            self.next_u[s] += 1
        return sub, u

    def batch(self, n_new, n_hit, fat=0, unique=False):
        """(sub, u, is_new) of one batch in random order: n_new new flows of the regular subscribers plus `fat` of FAT,
        and n_hit frames of flows made in the last three batches (each flow once when `unique`)."""
        sub, u = self.new(np.concatenate([self.r.integers(0, N_SUBS, n_new), np.full(fat, FAT)]))
        old_s = np.concatenate([b[0] for b in self.batches[-3:]]) if self.batches else np.zeros(0, np.int64)
        old_u = np.concatenate([b[1] for b in self.batches[-3:]]) if self.batches else np.zeros(0, np.int64)
        self.batches.append((sub, u))
        if n_hit and len(old_s):
            pick = self.r.choice(len(old_s), min(n_hit, len(old_s)), replace=not unique)
            sub, u = np.concatenate([sub, old_s[pick]]), np.concatenate([u, old_u[pick]])
        is_new = np.arange(len(sub)) < len(self.batches[-1][0])
        order = self.r.permutation(len(sub))
        return sub[order], u[order], is_new[order]

    def clock(self, n, per_frame):
        """(now, now_v): a clock value per frame, 1..4 us apart, or one for the batch."""
        if per_frame:
            now_v = (self.t + np.cumsum(self.r.integers(1_000, 4_000, n))).astype(np.uint64)
            self.t = int(now_v[-1]) + 10**6
            return int(now_v[0]), now_v
        self.t += 10**7
        now = self.t
        self.t += 10**7
        return now, None


def _rows(a) -> set:
    return {bytes(r) for r in np.asarray(a)}


def _port_host(b) -> int:
    return (int(b[0]) << 8) | int(b[1])


# ---------------------------------------------------------------------------
# the checker
# ---------------------------------------------------------------------------
class Replay:
    """The oracle (reference capacities: it never fills) next to a dataplane `dev` with small LRU tables, both loaded
    with the same maps; `batch` runs one batch on both and checks it."""

    def __init__(self, kind, dev, maps: harness.Script):
        self.ora = harness.OracleBackend(kind)
        self.o = self.ora.o
        self.dev = dev
        for st in maps.steps:
            assert self.ora.update(st[1], st[2], st[3], st[4]) == 0 and dev.update(st[1], st[2], st[3], st[4]) == 0, st[1]
        self.deleted = {m: 0 for m in LRU}
        self.victims = []  # nat_sessions keys the replay deleted
        self.log = []  # per batch: (prog, deletions per table, frames that hit a session older than the batch, frames out)

    def close(self):
        self.ora.close()

    def observe(self, prog, arena, lens, now, now_v):
        """Runs the batch on the device and takes everything observable."""
        a, ln = arena.copy(), lens.copy()
        v = self.dev.run(prog, a, ln, now, None, 64, None, now_v)
        got = {"verdict": np.asarray(v).copy(), "frames": a, "len": ln}
        got["events"] = {m: self.dev.drain(m) for m in harness.EVENT_MAPS}
        got["stats"] = {m: self.dev.stats(m) for m in harness.STATS_MAPS}
        got["dumps"] = {m: self.dev.dump(m) for m in harness.TABLES}
        got["info"] = {m: self.dev.map_info(m) for m in LRU}
        got["health"] = self.dev.health()
        return got

    def batch(self, prog, frames, now, now_v=None, corrupt=None):
        n = len(frames)
        arena, lens = frames.reshape(-1).copy(), np.full(n, 64, np.uint32)
        got = self.observe(prog, arena, lens, now, now_v)
        if corrupt is not None:
            corrupt(got, frames)
        return self.check(prog, frames, arena, lens, now, now_v, got)

    def check(self, prog, frames, arena, lens, now, now_v, got):
        o, n = self.o, len(frames)
        fail = []
        # ---- 1. the frame each SESSION_CREATE record came from ----
        ev = got["events"]["nat_log_rb"]
        rec = ev[ev[:, 8:12].copy().view("<u4").reshape(-1) == 1] if len(ev) else np.zeros((0, 40), np.uint8)
        if now_v is not None:
            where = {int(t): i for i, t in enumerate(now_v)}
            idx = [where.get(int(t), -1) for t in rec[:, 0:8].copy().view("<u8").reshape(-1)]
        else:
            tk = np.concatenate([frames[:, 26:30], frames[:, 30:34], frames[:, 34:36], frames[:, 36:38], frames[:, 23:24]], axis=1)
            where = {}
            for i, r in enumerate(tk):  # (a 5-tuple twice in one batch names no frame: -2)
                where[bytes(r)] = -2 if bytes(r) in where else i
            rk = np.concatenate([rec[:, 16:20], rec[:, 28:32], rec[:, 24:26], rec[:, 32:34], rec[:, 34:35]], axis=1)
            idx = [where.get(bytes(r), -1) for r in rk]
            assert -2 not in idx, "a record of a 5-tuple that comes twice in a single-clock batch"
            idx = [i if i >= 0 else -1 for i in idx]
        if -1 in idx:
            fail.append(f"  {idx.count(-1)} SESSION_CREATE records name no frame of the batch")
        creators = sorted((i, j) for j, i in enumerate(idx) if i >= 0)

        # ---- 2. the oracle, in index order, in segments split at the creating frames ----
        before = {m: int(o.map_info(m)["count"]) for m in LRU}
        dels = {m: 0 for m in LRU}
        oa = o.arena(len(arena) + 64)
        oa[:len(arena)] = arena
        ol = lens.copy()
        verdict = np.zeros(n, np.uint8)
        pos = 0

        def run_to(end):
            nonlocal pos
            if end > pos:
                verdict[pos:end] = o.run(prog, oa[pos * 64:end * 64], ol[pos:end], now, stride=64,
                                         now_v=None if now_v is None else now_v[pos:end])
                pos = end

        seen_before = _rows(o.dump("nat_sessions")[0])
        for i, j in creators:
            run_to(i)
            r = rec[j]
            key = np.zeros(16, np.uint8)
            key[0:4], key[4:8], key[8:10], key[10:12], key[12] = r[16:20], r[28:32], r[24:26], r[32:34], r[34]
            if o.lookup("nat_sessions", key) is not None:
                assert o.delete("nat_sessions", key) == 0
                dels["nat_sessions"] += 1
                self.victims.append(key)
            ek = np.zeros(8, np.uint8)
            ek[0:4], ek[4:6], ek[6] = r[16:20], r[24:26], r[34]
            m = o.lookup("eim_table", ek)
            if m is not None and (int(m[4]) | int(m[5]) << 8) != _port_host(r[26:28]):
                assert o.delete("eim_table", ek) == 0
                dels["eim_table"] += 1
        run_to(n)
        mid = dict(dels)
        end = {m: int(o.map_info(m)["count"]) for m in LRU}
        ora_ev = {m: self.ora.drain(m) for m in harness.EVENT_MAPS}
        ora_frames = oa[:len(arena)].copy()
        o.free_arenas()

        # ---- 3. reconcile the LRU tables ----
        for m in LRU:
            gk = _rows(got["dumps"][m][0])
            ok = o.dump(m)[0]
            for row in ok:
                if bytes(row) not in gk:
                    assert o.delete(m, row) == 0
                    dels[m] += 1
                    if m == "nat_sessions":
                        self.victims.append(row)
            extra = len(gk - _rows(o.dump(m)[0]))
            if extra:
                fail.append(f"  {m}: {extra} keys live on the device that the oracle does not hold")

        # ---- 4. bit for bit ----
        res_o = {"verdict": verdict, "len": ol, "frames": ora_frames}
        res_d = {"verdict": got["verdict"], "len": got["len"], "frames": got["frames"]}
        for m in harness.EVENT_MAPS:
            a, b = ora_ev[m], got["events"][m]
            res_o["ev_" + m] = harness.mask_padding(m, a) if len(a) else np.zeros((0, 1), np.uint8)
            res_d["ev_" + m] = harness.mask_padding(m, b) if len(b) else np.zeros((0, 1), np.uint8)
        for m in harness.STATS_MAPS:
            res_o["st_" + m], res_d["st_" + m] = self.ora.stats(m), got["stats"][m]
        for m in harness.TABLES:
            for res, (k, v) in ((res_o, self.ora.dump(m)), (res_d, got["dumps"][m])):
                res["tk_" + m] = k
                res["tv_" + m] = harness.mask_padding(m, v) if v.shape[0] else v
        fail += [f"  {k}: {msg}" for k, msg in harness.diff_keys(res_o, res_d)]

        # ---- 5. every deletion was needed, nothing refused or lost, the tables within their size ----
        for m in LRU:
            inserted = end[m] - before[m] + mid[m]
            cap = int(got["info"][m]["max_entries"])
            if dels[m] and before[m] + inserted <= cap:
                fail.append(f"  {m}: {dels[m]} entries gone in a batch that never filled it ({before[m]} live + {inserted} "
                            f"inserted <= {cap})")
            cnt, dl = int(got["info"][m]["count"]), len(got["dumps"][m][0])
            if not cnt == dl <= cap:
                fail.append(f"  {m}: count {cnt}, dump {dl}, max_entries {cap}")
        for k, v in got["health"].items():
            if v:
                fail.append(f"  {k} = {v}")
        if fail:
            raise AssertionError(f"{prog}, batch {len(self.log)}: {len(fail)} findings\n" + "\n".join(fail[:60]))
        for m in LRU:
            self.deleted[m] += dels[m]
        # frames that hit (no record) a session that existed before the batch
        tk = np.zeros((n, 16), np.uint8)
        tk[:, 0:4], tk[:, 4:8], tk[:, 8:12], tk[:, 12] = frames[:, 26:30], frames[:, 30:34], frames[:, 34:38], frames[:, 23]
        made = {i for i, _ in creators}
        old_hits = np.array([i not in made and bytes(tk[i]) in seen_before for i in range(n)], bool)
        self.log.append((prog, dels, old_hits, got["frames"].reshape(n, 64), got["verdict"]))
        return got


# ---------------------------------------------------------------------------
# the dataplanes: the device, and a fake one for checking the checker
# ---------------------------------------------------------------------------
class Device(harness.GpuBackend):
    def map_info(self, m):
        return self.dp.map_info(m)


class FakeDataplane(harness.OracleBackend):
    """A second oracle (a private copy of the library: its own map state) that keeps the LRU tables at the device's
    small sizes itself: a batch runs in segments that cannot overflow, and, once a table is full, frame by frame; when a
    frame's insert takes a table past its size, seeded-random victims other than what the frame itself used give way —
    entries made earlier in the same batch included.  Every run it makes is one the replay must accept."""

    def __init__(self, kind, tmpdir, seed, caps=None):
        from oracle import pyoracle
        src = pyoracle.REF_LIB if kind == "reference" else pyoracle.PORT_LIB
        path = os.path.join(str(tmpdir), "libfake_" + os.path.basename(src))
        shutil.copy(src, path)
        self.o, self.kind = pyoracle.Oracle(kind, path=path), "fake"
        self.caps = caps or {"nat_sessions": SES_CAP, "nat_reverse": SES_CAP, "eim_table": EIM_CAP}
        self.r = np.random.Generator(np.random.PCG64(seed))
        self.evicted = {m: 0 for m in LRU}

    def map_info(self, m):
        inf = self.o.map_info(m)
        inf["max_entries"] = self.caps[m]
        return inf

    def health(self):
        return {}

    def _count(self, m):
        return int(self.o.map_info(m)["count"])

    def _evict(self, m, over, keep):
        inf = self.o.map_info(m)
        keys = np.zeros((int(inf["count"]), inf["key_size"]), np.uint8)
        vals = np.zeros((len(keys), inf["value_size"]), np.uint8)
        n = self.o.lib.ora_map_dump(self.o.map_id(m), keys.ctypes.data, vals.ctypes.data, len(keys))
        pool = np.flatnonzero((keys[:n] != np.frombuffer(keep, np.uint8)).any(axis=1))
        for i in self.r.choice(pool, over, replace=False):
            assert self.o.delete(m, keys[i]) == 0
        self.evicted[m] += over

    def run(self, prog, arena, lens, now, off16, stride, prio, now_v=None):
        assert off16 is None and stride == 64 and prio is None
        n = len(lens)
        fr = arena.reshape(n, 64).copy()
        oa = self.o.arena(len(arena) + 64)
        oa[:len(arena)] = arena
        verdict = np.zeros(n, np.uint8)
        pos = 0
        while pos < n:
            room = min(self.caps[m] - self._count(m) for m in LRU)
            end = pos + (min(room, n - pos) if room > 0 else 1)
            verdict[pos:end] = self.o.run(prog, oa[pos * 64:end * 64], lens[pos:end], now, stride=64,
                                          now_v=None if now_v is None else now_v[pos:end])
            if room <= 0:  # one frame at a full table: whatever it inserted stays, somebody else goes
                f = fr[pos]
                key = np.zeros(16, np.uint8)
                key[0:4], key[4:8], key[8:12], key[12] = f[26:30], f[30:34], f[34:38], f[23]
                ek = np.zeros(8, np.uint8)
                ek[0:4], ek[4:6], ek[6] = f[26:30], f[34:36], f[23]
                rk = np.zeros(16, np.uint8)
                s = self.o.lookup("nat_sessions", key)
                if s is not None:
                    rk[0:4], rk[4:8], rk[8:10], rk[10:12], rk[12] = f[30:34], s[0:4], f[36:38], s[4:6], f[23]
                keep = {"nat_sessions": bytes(key), "eim_table": bytes(ek), "nat_reverse": bytes(rk)}
                for m in LRU:
                    over = self._count(m) - self.caps[m]
                    if over > 0:
                        self._evict(m, over, keep[m])
            pos = end
        arena[:] = oa[:len(arena)]
        self.o.free_arenas()
        return verdict


# ---------------------------------------------------------------------------
# workloads
# ---------------------------------------------------------------------------
PROGS = {"egress_eim": ("nat44_egress", 0x0F), "egress_noeim": ("nat44_egress", 0x0E), "pipeline_up": ("pipeline_up", 0x0F),
         "pipeline_tc": ("pipeline_tc", 0x0F)}
# (a) one batch of 3.5x the session table in new flows; (b) a full table, 80 % hits on older flows and 20 % new, and
# (d) the same with one clock per batch and each 5-tuple once per batch (the benchmark's mode: last_seen is
# epoch-stamped); (c) one subscriber with 600 new flows per batch among the others, over several 256-frame stages
SHAPES = ("flood", "churn", "fat", "churn_1clk")


def shape_batches(shape, tr):
    if shape == "flood":
        yield tr.batch(7168, 0)
    elif shape in ("churn", "churn_1clk"):
        yield tr.batch(2600, 0)
        for _ in range(9):
            yield tr.batch(500, 2000, unique=shape == "churn_1clk")
    else:
        yield tr.batch(2000, 0)
        for _ in range(8):
            yield tr.batch(300, 1200, fat=600)


def drive(rep, tr, prog, shape, batches=None):
    per_frame = shape != "churn_1clk"
    for b, (sub, u, _) in enumerate(shape_batches(shape, tr)):
        if batches is not None and b == batches:
            break
        fr = flow_frames(sub, u)
        now, now_v = tr.clock(len(fr), per_frame)
        rep.batch(prog, fr, now, now_v)


def replies(rep, tr, per_frame):
    """Replies to flows of every age — the first batch's and the last one's, evenly sampled — each twice or three
    times: DNAT, the stale-reverse path (sessions_expired) and replies whose reverse entry went."""
    outs = []
    for _, _, _, fr, vd in {id(b): b for b in (rep.log[0], rep.log[-1])}.values():
        fr = fr[vd == 0]
        outs.append(fr[::max(1, len(fr) // 1200)])
    out = np.concatenate(outs)
    rp = out.copy()
    rp[:, 26:30], rp[:, 30:34] = out[:, 30:34], out[:, 26:30]
    rp[:, 34:36], rp[:, 36:38] = out[:, 36:38], out[:, 34:36]
    rp[rp[:, 23] == 6, 47] = 0x10
    rp = np.concatenate([rp, rp, rp[::3]])
    rp = rp[tr.r.permutation(len(rp))]
    before = rep.ora.stats("nat_stats_map").copy()
    now, now_v = tr.clock(len(rp), per_frame)
    rep.batch("nat44_ingress", rp, now, now_v)
    d = rep.ora.stats("nat_stats_map") - before
    st = dict(zip(L.nat_stats.names, d))
    assert st["packets_dnat"] > 0 and st["sessions_expired"] > 0 and st["packets_passed"] > 0, st


def blocks_did_not_wrap(rep):
    k, v = rep.ora.dump("subscriber_nat")
    sn = v.view(L.subscriber_nat).reshape(-1)
    ports = sn["block"]["port_end"].astype(np.int64) - sn["block"]["port_start"] + 1
    assert (sn["sessions_total"].astype(np.int64) <= ports).all(), "a port block may have wrapped: the replay is not exact"


# ---------------------------------------------------------------------------
# the checker, on the CPU: legal eviction runs pass, corrupted ones do not
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["flood", "churn", "churn_1clk"])
@pytest.mark.parametrize("prog", ["egress_eim", "egress_noeim", "pipeline_tc"])
def test_replay_accepts_random_legal_evictions(shape, prog, lru_oracle, tmp_path):
    name, flags = PROGS[prog]
    fake = FakeDataplane(lru_oracle, tmp_path, seed=len(shape) * 7 + flags)
    rep = Replay(lru_oracle, fake, maps_script(flags, name))
    try:
        drive(rep, Traffic(0x1A0 + flags), name, shape, batches=4)
        for m in LRU:  # (a reverse entry the fake evicted may come back with a recreated session: nothing to delete)
            if m != "eim_table" or flags & 1:
                assert 0 < rep.deleted[m] <= fake.evicted[m], (m, rep.deleted, fake.evicted)
        blocks_did_not_wrap(rep)
    finally:
        rep.close()
        fake.close()


def _corrupt_port(got, frames):
    fr, vd = got["frames"].reshape(-1, 64), got["verdict"]
    ok = np.flatnonzero((vd == 0) & (fr[:, 26:30] != frames[:, 26:30]).any(axis=1))
    i = ok[0]
    j = next(j for j in ok[1:] if (fr[j, 34:36] != fr[i, 34:36]).any() and (frames[j, 26:30] != frames[i, 26:30]).any())
    fr[i, 34:36] = fr[j, 34:36]


def _bump(table, off, width):
    def corrupt(got, frames):
        k, v = got["dumps"][table]
        v = v.copy()
        i = len(v) // 2
        v[i, off:off + width] = np.frombuffer((int.from_bytes(v[i, off:off + width].tobytes(), "little") + 1)
                                              .to_bytes(width, "little"), np.uint8)
        got["dumps"][table] = (k, v)
    return corrupt


def _drop_record(got, frames):
    ev = got["events"]["nat_log_rb"]
    created = np.flatnonzero(ev[:, 8] == 1)
    got["events"]["nat_log_rb"] = np.delete(ev, created[len(created) // 2], axis=0)


def _extra_entry(got, frames):
    k, v = got["dumps"]["nat_sessions"]
    nk = k[:1].copy()
    nk[0, 10:12] = [0x1F, 0x90]  # destination port 8080: no flow of these workloads
    order = np.lexsort(np.concatenate([k, nk]).T[::-1])
    got["dumps"]["nat_sessions"] = (np.concatenate([k, nk])[order], np.concatenate([v, v[:1]])[order])
    got["info"]["nat_sessions"] = dict(got["info"]["nat_sessions"], count=len(k) + 1)


CORRUPTIONS = {
    "another_flows_port": _corrupt_port,
    "packet_on_a_foreign_session": _bump("nat_sessions", 40, 8),   # packets_out
    "foreign_eim_ref_count": _bump("eim_table", 24, 4),            # ref_count
    "survivor_last_seen_shifted": _bump("nat_sessions", 24, 8),    # last_seen
    "creation_record_missing": _drop_record,
    "extra_live_entry": _extra_entry,
}


@pytest.mark.parametrize("what", CORRUPTIONS)
def test_replay_rejects_a_corrupted_run(what, lru_oracle, tmp_path):
    """A legal run of the fake dataplane passes its first batch; the second — hits on old sessions, new flows and
    evictions — passes too, except with one corruption of what the dataplane shows."""
    name, flags = PROGS["egress_eim"]
    fake = FakeDataplane(lru_oracle, tmp_path, seed=0xC0)
    rep = Replay(lru_oracle, fake, maps_script(flags, name))
    try:
        tr = Traffic(0x1C0)
        batches = shape_batches("churn", tr)
        sub, u, _ = next(batches)
        fr = flow_frames(sub, u)
        rep.batch(name, fr, *tr.clock(len(fr), True))
        sub, u, _ = next(batches)
        fr = flow_frames(sub, u)
        now, now_v = tr.clock(len(fr), True)
        with pytest.raises(AssertionError):
            rep.batch(name, fr, now, now_v, corrupt=CORRUPTIONS[what])
        assert all(fake.evicted[m] > 0 for m in LRU)
    finally:
        rep.close()
        fake.close()


# ---------------------------------------------------------------------------
# the device
# ---------------------------------------------------------------------------
FEEDS = {"pageable": False, "pinned": True, "device": "device"}


def sweep_matches(rep, now):
    """bng_sweep against sweep_spec on the reconciled oracle: evictions are silent, so EIM reference counts stay above
    the live sessions that use them, and the sweep must agree on what that leaves."""
    want = sweep_spec(rep.o, now)
    n = rep.dev.dp.sweep(now)
    got = rep.dev.dp.drain("nat_log_rb")
    assert n == len(want), f"sweep at {now // NS} s: {n} sessions removed, the spec says {len(want)}"
    if n:
        assert np.array_equal(harness.mask_padding("nat_log_rb", got), harness.mask_padding("nat_log_rb", want)), \
            f"sweep at {now // NS} s: SESSION_DELETE records differ"
    for m in SWEEP_MAPS:
        (ok, ov), (gk, gv) = rep.ora.dump(m), rep.dev.dump(m)
        assert np.array_equal(ok, gk), f"sweep at {now // NS} s: {m} keys differ"
        if len(ov):
            assert np.array_equal(harness.mask_padding(m, ov), harness.mask_padding(m, gv)), f"sweep at {now // NS} s: {m} differs"
    assert np.array_equal(rep.ora.stats("nat_stats_map"), rep.dev.stats("nat_stats_map")), f"sweep at {now // NS} s: stats"
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("feed", FEEDS)
@pytest.mark.parametrize("prog", PROGS)
@pytest.mark.parametrize("shape", SHAPES)
def test_full_flow_tables_match_the_oracle(shape, prog, feed, lru_oracle, monkeypatch):
    """Every batch with the device's evictions replayed on the oracle, bit for bit; then replies through
    nat44_ingress, the port-usage census over the device's tables and bng_sweep at two times."""
    if feed == "pinned":
        monkeypatch.setenv("BNG_ZC_CHUNK_LOG2", "10")  # read by bng_open: batches cross chunks
    name, flags = PROGS[prog]
    t0 = time.perf_counter()
    dev = Device(pinned=FEEDS[feed], max_subscribers=1 << 10, max_nat_sessions=SES_CAP, max_eim_mappings=EIM_CAP,
                 max_batch=1 << 14)
    rep = Replay(lru_oracle, dev, maps_script(flags, name))
    try:
        assert all(dev.map_info(m)["max_entries"] == (EIM_CAP if m == "eim_table" else SES_CAP) for m in LRU)
        rebuilds0 = dev.dp.table_rebuilds
        tr = Traffic(0x1E0 + 16 * SHAPES.index(shape) + flags)
        drive(rep, tr, name, shape)
        blocks_did_not_wrap(rep)
        per_frame = shape != "churn_1clk"
        rebuilds = dev.dp.table_rebuilds - rebuilds0
        evictions = dev.dp.lru_evictions
        for m in LRU:
            if m != "eim_table" or flags & 1:
                assert rep.deleted[m] > 0, f"{m}: the replay deleted nothing ({rep.deleted})"
        if not flags & 1:
            assert dev.map_info("eim_table")["count"] == 0
        if shape in ("churn", "churn_1clk"):
            assert rebuilds > 0, f"{evictions} evictions and no rebuild of the flow tables"
        if shape == "fat":
            fat_ip = bytes(S.ip_bytes(S.sub_ip(np.array([FAT])))[0])
            assert sum(bytes(k[0:4]) == fat_ip for k in rep.victims) > 0, "none of the fat subscriber's flows gave way"
        if shape == "churn" and name == "pipeline_tc":
            # frames of subscribers with a bucket run all of nat44_egress in the ordered phase; some of them hit
            # sessions older than their batch in batches that evicted
            deferred_old = 0
            for _, dels, old_hits, fr, _ in rep.log[1:]:
                if dels["nat_sessions"]:
                    sub = (fr[:, 26:30].copy().view(">u4").reshape(-1) - 0x64400000) & 0xFFFF
                    deferred_old += int((old_hits & (sub % 2 == 0)).sum())
            assert deferred_old > 0
        census = check_census(dev.dp, {m: dev.dump(m) for m in ("subscriber_nat", "nat_sessions", "eim_table", "nat_reverse")},
                              f"{shape} {prog} {feed}")
        assert census[0]["unreachable"] > 0, census[0]
        replies(rep, tr, per_frame)
        swept = sweep_matches(rep, tr.t + 130 * NS) + sweep_matches(rep, tr.t + 300 * NS)
        assert swept > 0
        assert dev.dp.lru_overflow == 0 and dev.dp.events_lost == 0
        print(f"\n[lru] {shape} {prog} {feed}: replay deletions {rep.deleted}, lru_evictions {evictions}, "
              f"table_rebuilds {rebuilds}, batches {len(rep.log)}, {time.perf_counter() - t0:.1f} s")
    finally:
        rep.close()
        dev.close()
