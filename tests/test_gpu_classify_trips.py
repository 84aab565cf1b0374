"""k_pipe_classify is a persistent grid-stride loop, one frame per lane: its grid is SMs x the blocks per SM it is
compiled for, and a warp reads its 32 headers 64 bytes wide only when every active lane's frame allows it.  These
scripts put the batch end where warps of one launch make different numbers of trips (grid x 256 +-1 and +-32 frames,
and a batch of three trips), make wide and 16-byte-chunk warp-trips alternate inside one batch, pack short frames back
to back so that a 64-byte window covers the next frame, and end the arena right behind the last header or one granule
after it.  All three classify instantiations (nat44_egress, pipeline_up, pipeline_tc) are compared with the CPU oracle,
bit for bit, on every feed."""
import os
import re

import numpy as np
import pytest

import harness
import scenarios
from harness import Script
from test_oracle_fuzz import TARGETS, base_maps_and_frames

pytestmark = pytest.mark.gpu
FEEDS = {"pageable": False, "pinned": True, "device": "device"}
PROGS = ["nat44_egress", "pipeline_up", "pipeline_tc"]
MS = 1_000_000
BLOCK = 256
SHORT = np.array([20, 34, 38, 42, 48, 50, 54, 60], np.uint32)
CLASSIFY_SRC = os.path.join(os.path.dirname(__file__), "..", "bng_b200", "csrc", "pipe_classify.cuh")


def classify_grid(prog):
    """Blocks of the classify launch at a large batch: SMs x the blocks per SM the kernel is compiled for, which is
    read from pipe_classify.cuh.  A library loaded through BNG_B200_LIB may have been built from other sources, whose
    trip edges lie elsewhere, so the test does not claim to check those edges there."""
    import torch
    from bng_b200 import dataplane
    if os.path.realpath(dataplane.LIB_PATH) != os.path.realpath(os.path.join(dataplane.HERE, "libbng_b200.so")):
        pytest.skip(f"trip edges follow the in-tree build's blocks per SM; BNG_B200_LIB = {dataplane.LIB_PATH}")
    src = open(CLASSIFY_SRC).read()
    name = "CLASSIFY_BLOCKS_NAT" if prog == "nat44_egress" else "CLASSIFY_BLOCKS"
    bps = int(re.search(rf"#define {name} (\d+)", src).group(1))
    return torch.cuda.get_device_properties(0).multi_processor_count * bps


def mixed_layout(lens, tail_room):
    """off16 for frames placed so that warp-trips (32 consecutive frames) alternate between all 32-byte aligned
    (read wide) and not (lane 0 sits 16 bytes off a 32-byte boundary), each frame in ceil(len / 16) granules right
    behind the previous one, so a short frame's 64-byte window reaches into its neighbour.  The last group is
    read wide, and the arena ends `tail_room` bytes after the start of the last frame."""
    n = len(lens)
    off = np.zeros(n, np.int64)
    cur = 0
    last_group = (n - 1) // 32
    for j in range(n):
        g = j // 32
        if (last_group - g) % 2 == 0:
            cur = (cur + 31) // 32 * 32
        else:
            cur = (cur + 15) // 16 * 16
            if j % 32 == 0 and cur % 32 == 0:
                cur += 16
        off[j] = cur
        cur += (int(lens[j]) + 15) // 16 * 16
    return off, int(off[-1]) + tail_room


def trips_script(prog, grid):
    updates, frames, lens0, now, _ = base_maps_and_frames(TARGETS[prog])
    frames = np.ascontiguousarray(frames[:, :64])
    r = scenarios.rng(0x57A6 + len(prog))
    edge = grid * BLOCK
    sc = Script(f"classify_trips_{prog}")
    sc.steps = list(updates)
    pos = 0

    def take(n):
        nonlocal pos
        idx = np.arange(pos, pos + n) % len(frames)
        pos += n
        lens = np.minimum(lens0[idx], 128).astype(np.uint32)
        short = r.random(n) < 0.3
        lens[short] = r.choice(SHORT, int(short.sum()))
        return frames[idx], lens

    # a fixed-stride ring whose last frame's 64 bytes end exactly at the end of the arena
    f, l = take(edge + 1)
    sc.run(prog, f.reshape(-1).copy(), l, now + 1, stride=64)
    sc.drain()
    # offset tables: the batch ends at +-1 and +-32 frames of one trip per warp, and one batch takes three trips;
    # the last frame is 64 bytes long and the arena (whole 16-byte granules) ends one granule past it, the least room
    # in which its header is still read wide (the kernels may touch arena_bytes * 16 - 15 bytes), or right at its end
    # (read in 16-byte chunks)
    for b, (n, tail) in enumerate([(edge - 32, 80), (edge - 1, 64), (edge + 1, 80), (edge + 32, 64), (2 * edge + 33, 80)]):
        f, l = take(n)
        l[-1] = 64
        off, total = mixed_layout(l, tail)
        arena = np.zeros(total, np.uint8)
        keep = np.arange(64)[None, :] < np.minimum(l, 64)[:, None]
        arena[(off[:, None] + np.arange(64)[None, :])[keep]] = f[keep]
        sc.run(prog, arena, l, now + (b + 2) * MS, off16=(off // 16).astype(np.uint32))
        sc.drain()
    return sc


_oracle = {}


@pytest.mark.parametrize("feed", list(FEEDS))
@pytest.mark.parametrize("prog", PROGS)
def test_classify_trips_against_oracle(prog, feed, ora_kind):
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    grid = classify_grid(prog)
    key = (prog, ora_kind, grid)
    if key not in _oracle:
        _oracle[key] = harness.run_script(harness.OracleBackend(ora_kind), trips_script(prog, grid))
    # room for a whole batch and for its events (drained after every batch)
    be = harness.GpuBackend(pinned=FEEDS[feed], max_batch=1 << 19, event_capacity=1 << 19)
    try:
        got = harness.run_script(be, trips_script(prog, grid))
    finally:
        be.close()
    harness.compare(_oracle[key], got, f"classify trips {prog} ({feed}): {ora_kind} oracle vs gpu")
