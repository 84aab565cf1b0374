"""Batch, tile and ring boundaries against the CPU oracle, bit for bit, on all three ways of feeding a batch.

The kernels work in tiles: classify blocks of 256 frames, a resolve stage of 256 frames of one subscriber (a warp
times RS_PER_THREAD), radix-scatter tiles of 2048 frames, DHCP TMA tiles of 128 frames and zero-copy chunks of
BNG_ZC_CHUNK_LOG2 frames.  Off-by-one errors live at the ends of those tiles, so the scripts here put the end of a
batch, or the end of one subscriber's run of frames, at +-1 of each of them."""
import numpy as np
import pytest

import harness
import scenarios
from bng_b200 import layouts as L
from bng_b200 import synth as S
from harness import Script
from test_oracle_fuzz import TARGETS, base_maps_and_frames

pytestmark = pytest.mark.gpu
FEEDS = {"pageable": False, "pinned": True, "device": "device"}
BATCH_SIZES = [1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 2047, 2048, 2049]
MS = 1_000_000


def _cached(fn):
    cache = {}

    def get(*key):
        if key not in cache:
            cache[key] = fn(*key)
        return cache[key]

    return get


def _run(be, script):
    try:
        return harness.run_script(be, script)
    finally:
        be.close()


def _add_batch(sc, prog, frames, lens, now, packed):
    """One run of frames u8[n, w]: through an offset table when the scenario's corpus is variable-length."""
    if packed:
        arena, off16 = S.pack_arena(frames, lens)
        sc.run(prog, arena, lens, now, off16=off16)
    else:
        sc.run(prog, frames.reshape(-1).copy(), lens, now, stride=frames.shape[1])


def _scenario_frames(prog):
    updates, frames, lens, now, _ = base_maps_and_frames(TARGETS[prog])
    if prog == "qos_egress_prog":  # the corpus is upload traffic: swap the addresses so the download buckets apply
        frames = frames.copy()
        frames[:, 26:30], frames[:, 30:34] = frames[:, 30:34].copy(), frames[:, 26:30].copy()
    packed = next(st for st in scenarios.ALL_SCRIPTS[TARGETS[prog]]().steps if st[0] == "run")[5] is not None
    return updates, frames, lens, now, packed


def batch_edges_script(prog, sizes=BATCH_SIZES, drain_after=6):
    """The scenario's maps, then its frames (repeated as needed) cut into consecutive batches of `sizes` frames,
    each with its own clock, and one drain of the event rings in the middle."""
    updates, frames, lens, now, packed = _scenario_frames(prog)
    sc = Script(f"edges_{prog}")
    sc.steps = list(updates)
    pos = 0
    for b, n in enumerate(sizes):
        idx = np.arange(pos, pos + n) % len(frames)
        pos += n
        _add_batch(sc, prog, frames[idx], lens[idx].copy(), now + b * MS + 1, packed)
        if b == drain_after:
            sc.drain()
    return sc


_oracle_edges = _cached(lambda prog, kind: harness.run_script(harness.OracleBackend(kind), batch_edges_script(prog)))


@pytest.mark.parametrize("feed", list(FEEDS))
@pytest.mark.parametrize("prog", sorted(TARGETS))
def test_batch_edges_against_oracle(prog, feed, ora_kind):
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    got = _run(harness.GpuBackend(pinned=FEEDS[feed]), batch_edges_script(prog))
    harness.compare(_oracle_edges(prog, ora_kind), got, f"batch edges {prog} ({feed}): {ora_kind} oracle vs gpu")


# ---------------------------------------------------------------------------
# one subscriber's run of frames at the edges of the resolve stage (256 frames) and of the chain of warps
# ---------------------------------------------------------------------------
SUB_RUNS = [255, 256, 257, 511, 512, 513]
SUB_RUN_PROGS = ["qos_ingress_prog", "qos_egress_prog", "pipeline_up", "pipeline_tc", "nat44_egress"]
N_SUBS, FAT, OTHERS = 24, 5, 700


def sub_runs_script(prog):
    """Each batch: OTHERS frames of mixed traffic from every subscriber but FAT, and exactly K frames of subscriber
    FAT at random positions among them, K in SUB_RUNS.  FAT's frames are all new flows (a fresh source port each,
    in a port block of 4096), so nat44_egress / the pipelines create K sessions of one subscriber in one batch; its
    buckets let about 256 64-byte frames through, so the token bucket turns from pass to drop inside the run."""
    r = scenarios.rng(0xB0D7 + len(prog))
    sc = Script(f"subrun_{prog}")
    keys, v = S.bindings(N_SUBS)
    sc.update("subscriber_bindings", keys, v)
    cfg = np.zeros(1, L.antispoof_config)
    cfg["default_mode"], cfg["log_violations"] = 1, 1
    sc.update1("antispoof_config", np.uint32(0), cfg)
    pubs = scenarios.nat_maps(sc, N_SUBS, 4096, 0x0F)
    for m in ("qos_ingress", "qos_egress"):
        qk, qv = S.qos_buckets(N_SUBS, upload=m == "qos_ingress")
        qv["rate_bps"][FAT], qv["burst_bytes"][FAT] = 8_000_000, 256 * 64 + 32
        qv["tokens"][FAT] = qv["burst_bytes"][FAT]
        sc.update(m, qk, qv)
    t = 10**9
    for b, k in enumerate(SUB_RUNS):
        hdr, lens = scenarios.nat_frames(r, N_SUBS, OTHERS, pubs)
        hdr[(hdr[:, 26:30] == S.ip_bytes(S.sub_ip(FAT))).all(axis=1), 29] ^= 0x40  # FAT sends nothing else
        proto = r.choice(np.array([6, 17], np.uint32), k)
        sport = (30000 + 600 * b + np.arange(k)).astype(np.uint32)
        flen = r.choice(np.array([64, 64, 64, 128, 594], np.uint32), k)
        fat = S.ipv4_headers(S.sub_mac_key(FAT), np.uint64(scenarios.GW_MAC), S.sub_ip(FAT),
                             (0x08080800 + r.integers(0, 4, k)).astype(np.uint32), proto, sport, 443, flen)
        n = OTHERS + k
        at = np.sort(r.choice(n, k, replace=False))
        rest = np.setdiff1d(np.arange(n), at)
        frames = np.zeros((n, 64), np.uint8)
        fl = np.zeros(n, np.uint32)
        frames[at], fl[at] = fat, flen
        frames[rest], fl[rest] = hdr, lens
        if prog == "qos_egress_prog":  # download traffic: the subscriber is the destination
            frames[:, 26:30], frames[:, 30:34] = frames[:, 30:34].copy(), frames[:, 26:30].copy()
        sc.run(prog, frames.reshape(-1).copy(), fl, t + b * MS, stride=64)
        if b == 2:
            sc.drain()
    return sc


_oracle_runs = _cached(lambda prog, kind: harness.run_script(harness.OracleBackend(kind), sub_runs_script(prog)))


@pytest.mark.parametrize("feed", list(FEEDS))
@pytest.mark.parametrize("prog", SUB_RUN_PROGS)
def test_subscriber_runs_against_oracle(prog, feed, ora_kind):
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    want = _oracle_runs(prog, ora_kind)
    got = _run(harness.GpuBackend(pinned=FEEDS[feed]), sub_runs_script(prog))
    harness.compare(want, got, f"subscriber runs {prog} ({feed}): {ora_kind} oracle vs gpu")
    # the runs did what they are for: FAT's flows were created in one go, its bucket ran dry in mid-run
    if prog in ("nat44_egress", "pipeline_up"):
        assert want["st_nat_stats_map"][5] >= sum(SUB_RUNS)
    if prog != "nat44_egress":
        assert want["st_qos_stats_map"][1] > 0


# ---------------------------------------------------------------------------
# zero-copy chunks: the pinned feed in chunks of 2^10 frames
# ---------------------------------------------------------------------------
ZC_SIZES = [1023, 1024, 1025, 3073]


@pytest.mark.parametrize("prog", ["nat44_egress", "dhcp_fastpath_prog"])
def test_zero_copy_chunk_edges_against_oracle(prog, ora_kind, monkeypatch):
    """nat44_egress on a 64-byte fixed-stride ring (copied as it is) and DHCP through an offset table (gathered and
    scattered by kernels): batches that end at +-1 of a chunk, and one that takes both chunk buffers twice."""
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    monkeypatch.setenv("BNG_ZC_CHUNK_LOG2", "10")  # read by bng_open
    want = harness.run_script(harness.OracleBackend(ora_kind), batch_edges_script(prog, ZC_SIZES, drain_after=1))
    got = _run(harness.GpuBackend(pinned=True), batch_edges_script(prog, ZC_SIZES, drain_after=1))
    harness.compare(want, got, f"zero-copy chunks of 1024 frames, {prog}: {ora_kind} oracle vs gpu")
