"""What translating inbound ICMP errors (bng_nat_icmp_errors_enable) costs nat44_ingress: the nat_ingress_64 workload
(replies to 1 M pre-created flows) at 2^22 frames, device-resident, the settings alternated in one process over several
rounds:
    off       translation off (k_nat_ingress)
    on_e0     translation on, no ICMP error frames (k_nat_ingress<icmperr>)
    on_e1     translation on, about 1 % of the frames replaced by ICMP errors quoting the workload's own flows
    on_e10    the same, about 10 %
An error is a Destination Unreachable (port unreachable, or fragmentation needed with an MTU of 1492) from a router
to the flow's public address, quoting the IPv4 header and first 8 bytes of the flow's SNATed frame: 70 bytes.  Every
setting uses the same layout: 128-byte slots, so that the error frames' quoted ports are present.  `off_64` is the
workload as bench.py stages it (64-byte slots), for reference.

The same four settings are then run from pinned host memory (BNG_MEM_HOST, the zero-copy feed): with the switch on,
nat44_ingress's header gather is k_gather_frames<true>, which also moves bytes 64-79 of the error frames.  These are
host-clock times of whole bng_prog_run calls (gather, program, scatter, verdict copy; the call synchronises).

    python tools/nat_icmp_cost.py [--steps 10] [--rounds 3] [--out FILE]

Prints one JSON document: the card (name, power limit, SM clock read after the runs), Mpps per round and setting, the
k_nat_ingress time of a profiled pass per setting (device events, bng_prof_*), the DNAT count of one batch, and the
pinned feed's ms per call per round and setting."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from li_cost import Rig, card  # noqa: E402
from qos_v6_cost import sm_clock  # noqa: E402

SETTINGS = ("off_64", "off", "on_e0", "on_e1", "on_e10")
ROUTER = (192, 0, 2, 1)


def with_errors(replies, snat, flow, share, seed, S):
    """replies (u8[n, 64]) widened to 128 bytes, a share of them replaced by errors quoting flow[i]'s SNATed frame."""
    n = replies.shape[0]
    out = np.zeros((n, 128), np.uint8)
    out[:, :64] = replies
    lens = np.full(n, 64, np.uint32)
    if not share:
        return out, lens
    r = np.random.default_rng(seed)
    idx = np.nonzero(r.random(n) < share)[0]
    q = snat[flow[idx]]
    f = np.zeros((len(idx), 128), np.uint8)
    f[:, 0:6], f[:, 6:12] = q[:, 6:12], q[:, 0:6]
    f[:, 12], f[:, 14], f[:, 17], f[:, 22], f[:, 23] = 0x08, 0x45, 56, 64, 1
    f[:, 26:30] = ROUTER
    f[:, 30:34] = q[:, 26:30]
    f[:, 24:26] = S.ip_checksum(f[:, 14:34])
    frag = r.random(len(idx)) < 0.5
    f[:, 34], f[:, 35] = 3, np.where(frag, 4, 3)
    f[frag, 40:42] = (0x05, 0xD4)  # next-hop MTU 1492
    f[:, 42:70] = q[:, 14:42]
    out[idx] = f
    lens[idx] = 70
    return out, lens


def pinned_cost(rigs, staged, rounds, torch, steps=5):
    """ms per bng_prog_run of each 128-byte-slot setting fed from pinned host memory (the zero-copy gather)."""
    from bng_b200 import MEM_HOST
    n = next(iter(staged.values()))[1].shape[0]
    ta = torch.zeros(n * 128, dtype=torch.uint8).pin_memory()  # one pinned arena, refilled before every call
    tv = torch.zeros(n, dtype=torch.uint8).pin_memory()
    feeds = {s: (torch.from_numpy(np.ascontiguousarray(h).reshape(-1)), torch.from_numpy(l.view(np.int32)).pin_memory())
             for s, (h, l) in staged.items()}
    out = {s: [] for s in staged}

    def run(s, k):
        r, (a0, tl) = rigs[s], feeds[s]
        ms = 0.0
        for _ in range(k):
            ta.copy_(a0)  # the frames as they arrive: each run DNATs them in place
            r.dp.sync()
            t0 = time.perf_counter()
            r.dp.run(r.wl.prog, ta, tl, r.wl.now0 + r.step_no * r.wl.now_step, stride=128, verdict=tv, mem=MEM_HOST,
                     arena_bytes=ta.numel())
            ms += (time.perf_counter() - t0) * 1e3
            r.step_no += 1
        return ms / k

    for s in staged:  # warm up
        run(s, 2)
    for _ in range(rounds):
        for s in staged:
            out[s].append(round(run(s, steps), 3))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=1 << 22)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from bng_b200 import layouts as L
    from bng_b200 import synth as S
    from bng_b200 import workloads as W
    dev = torch.device("cuda")
    res = {"card": card(), "workload": "nat_ingress_64", "frames": a.frames, "mpps": {s: [] for s in SETTINGS},
           "kernel_ms": {}, "dnat_per_batch": {}, "errors_per_batch": {}}
    rigs = {}
    for s in SETTINGS:
        wl = W.build("nat_ingress_64", a.frames, 0, 1, 1)
        rigs[s] = Rig(wl, torch, dev)
    base = rigs["off"]
    replies, lens64 = base.wl.derive(base.translated)
    snat = base.translated[0].reshape(-1, 64)
    # the flow each reply answers: derive() picks rows of the prewarm batch
    t = snat.copy()
    t[:, 26:30], t[:, 30:34] = snat[:, 30:34], snat[:, 26:30]
    flow = W._pick(0xB2000003 + 19, a.frames, snat.shape[0])
    assert (t[flow, 26:34] == replies[:, 26:34]).all(), "the replies' flows are not the prewarm rows"
    staged = {}
    for s, r in rigs.items():
        if s == "off_64":
            r.stage(replies, lens64)
        else:
            share = {"on_e1": 0.01, "on_e10": 0.10}.get(s, 0.0)
            h, l = with_errors(replies, snat, flow, share, 7, S)
            r.stage(h, l)
            staged[s] = (h, l)
            res["errors_per_batch"][s] = int((l == 70).sum())
        if s.startswith("on"):
            r.dp.nat_icmp_errors_enable(True)
    for s in SETTINGS:  # warm up every setting
        rigs[s].timed(2)
    for _ in range(a.rounds):
        for s in SETTINGS:
            mpps, _ = rigs[s].timed(a.steps)
            res["mpps"][s].append(round(mpps, 1))
    dnat = list(L.nat_stats.names).index("packets_dnat")
    for s in SETTINGS:
        r = rigs[s]
        r.dp.prof_enable(True)
        d0 = int(r.dp.stats("nat_stats_map")[dnat])
        for _ in range(5):
            r.restore()
            r.step()
            r.dp.sync()
        res["dnat_per_batch"][s] = (int(r.dp.stats("nat_stats_map")[dnat]) - d0) // 5
        prof = r.dp.prof_read()
        r.dp.prof_enable(False)
        r.restore()
        res["kernel_ms"][s] = {k: round(v[1] / v[0], 4) for k, v in prof.items() if "nat_ingress" in k}
    res["pinned_ms_per_call"] = pinned_cost(rigs, staged, a.rounds, torch)
    for r in rigs.values():
        r.dp.close()
    res["card"].update(sm_clock())
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
