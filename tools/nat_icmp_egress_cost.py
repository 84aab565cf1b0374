"""What translating subscribers' ICMP errors (bng_nat_icmp_errors_egress_enable) costs nat44_egress and pipeline_up:
the nat_steady_64 and pipeline_imix workloads at 2^22 frames, device-resident, the settings alternated in one process
over several rounds:
    off       translation off
    on_e0     translation on, no ICMP error frames (the ICMPERR instantiations of classify and resolve)
    on_e1     translation on, about 1 % of the frames replaced by subscriber errors
    on_e10    the same, about 10 %
An error replaces a subscriber's frame of the workload: a Destination Unreachable (port unreachable, or fragmentation
needed with an MTU of 1492) from the subscriber to the remote, quoting the IPv4 header and first 8 bytes of the remote's
reply to that flow as the subscriber received it (the workload's own inbound flow): 70 bytes.  Every setting uses the
same layout (headers staged 128 bytes wide), so that the error frames' quoted ports are present.

nat_steady_64 is then run from pinned host memory (BNG_MEM_HOST, the zero-copy feed): with the switch on the header
gather is k_gather_frames<true>, which also moves bytes 64-79 of the error frames.  These are host-clock times of whole
bng_prog_run calls.

    python tools/nat_icmp_egress_cost.py [--steps 10] [--rounds 3] [--out FILE]

Prints one JSON document: the card (name, power limit, SM clock read after the runs), Mpps per workload, round and
setting, the classify and resolve times of a profiled pass per setting (device events, bng_prof_*), the SNAT count of
one batch, and the pinned feed's ms per call per round and setting."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from li_cost import Rig, card  # noqa: E402
from nat_icmp_cost import pinned_cost  # noqa: E402
from qos_v6_cost import sm_clock  # noqa: E402

SETTINGS = ("off", "on_e0", "on_e1", "on_e10")
WORKLOADS = ("nat_steady_64", "pipeline_imix")


def with_errors(headers, lens, share, seed, S):
    """headers (u8[n, 64]) widened to 128 bytes, a share of the private-source IPv4 frames replaced by the sending
    subscriber's error about the remote's reply to that frame's flow."""
    n = headers.shape[0]
    out = np.zeros((n, 128), np.uint8)
    out[:, :64] = headers
    lens = lens.copy()
    if not share:
        return out, lens
    r = np.random.default_rng(seed)
    h = headers
    ok = (h[:, 12] == 8) & (h[:, 13] == 0) & (h[:, 14] == 0x45) & (h[:, 26] == 100) & np.isin(h[:, 23], (1, 6, 17))
    idx = np.nonzero(ok & (r.random(n) < share))[0]
    q = h[idx]
    rep = q.copy()  # the remote's reply as the subscriber received it
    rep[:, 26:30], rep[:, 30:34] = q[:, 30:34], q[:, 26:30]
    tu = q[:, 23] != 1
    rep[tu, 34:36], rep[tu, 36:38] = q[tu, 36:38], q[tu, 34:36]
    rep[~tu, 34] = 0
    f = np.zeros((len(idx), 128), np.uint8)
    f[:, 0:12] = q[:, 0:12]
    f[:, 12], f[:, 14], f[:, 17], f[:, 22], f[:, 23] = 0x08, 0x45, 56, 64, 1
    f[:, 26:30], f[:, 30:34] = q[:, 26:30], q[:, 30:34]
    f[:, 24:26] = S.ip_checksum(f[:, 14:34])
    frag = r.random(len(idx)) < 0.5
    f[:, 34], f[:, 35] = 3, np.where(frag, 4, 3)
    f[frag, 40:42] = (0x05, 0xD4)  # next-hop MTU 1492
    f[:, 42:70] = rep[:, 14:42]
    out[idx] = f
    lens[idx] = 70
    return out, lens


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
    snat = list(L.nat_stats.names).index("packets_snat")
    res = {"card": card(), "frames": a.frames, "mpps": {}, "kernel_ms": {}, "snat_per_batch": {}, "errors_per_batch": {},
           "pinned_ms_per_call": {}}
    for wname in WORKLOADS:
        rigs, staged = {}, {}
        for s in SETTINGS:
            wl = W.build(wname, a.frames, 0, 1, 1)
            r = rigs[s] = Rig(wl, torch, dev)
            if wl.derive is not None:
                wl.headers, wl.lens = wl.derive(r.translated)
            share = {"on_e1": 0.01, "on_e10": 0.10}.get(s, 0.0)
            h, l = with_errors(wl.headers, wl.lens, share, 7, S)
            r.stage(h, l)
            staged[s] = (h, l)
            res["errors_per_batch"][f"{wname}/{s}"] = int((l == 70).sum()) if share else 0
            if s.startswith("on"):
                r.dp.nat_icmp_errors_egress_enable(True)
        for s in SETTINGS:  # warm up every setting
            rigs[s].timed(2)
        res["mpps"][wname] = {s: [] for s in SETTINGS}
        for _ in range(a.rounds):
            for s in SETTINGS:
                mpps, _ = rigs[s].timed(a.steps)
                res["mpps"][wname][s].append(round(mpps, 1))
        for s in SETTINGS:
            r = rigs[s]
            r.dp.prof_enable(True)
            d0 = int(r.dp.stats("nat_stats_map")[snat])
            for _ in range(5):
                r.restore()
                r.step()
                r.dp.sync()
            res["snat_per_batch"][f"{wname}/{s}"] = (int(r.dp.stats("nat_stats_map")[snat]) - d0) // 5
            prof = r.dp.prof_read()
            r.dp.prof_enable(False)
            r.restore()
            res["kernel_ms"][f"{wname}/{s}"] = {k: round(v[1] / v[0], 4) for k, v in prof.items()}
        if wname == "nat_steady_64":  # (the imix layout goes through an offset table: not fed from pinned memory here)
            res["pinned_ms_per_call"][wname] = pinned_cost(rigs, staged, a.rounds, torch)
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
