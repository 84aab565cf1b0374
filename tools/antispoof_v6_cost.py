"""What letting a binding's own delegated prefixes count as its IPv6 addresses (bng_antispoof_ipv6_prefixes_enable)
costs the device-resident step: pipeline_imix (pipeline_up) and antispoof_64 (antispoof_ingress) at 2^22 frames, with
10 k subscribers x 2 prefixes (a /64 and a delegated /56, tools/dualstack_cost.py) installed in every setting, the flag
off and on alternated in one process over several rounds:
    off_p0 / on_p0    no IPv6 frames
    off_p20 / on_p20  about 20 % of the frames turned into IPv6 frames from hosts inside the sending subscriber's
                      delegated /56 (not from its binding's address, which the workloads leave unset)
    off_p50 / on_p50  the same, about 50 %
With the flag off those IPv6 frames are antispoof drops (strict mode), with it on they pass, so step rates do not
compare across off and on; kernel times do.

    python tools/antispoof_v6_cost.py [--steps 10] [--rounds 3] [--out FILE]

Prints one JSON document: the card (name, power limit, SM clock read after the runs), Mpps per round and setting,
frames dropped per batch, and the k_pipe_classify* / k_antispoof* kernel times of a profiled pass per setting (device
events, bng_prof_*)."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from dualstack_cost import N_SUBS, prefixes  # noqa: E402
from li_cost import Rig, card  # noqa: E402
from qos_v6_cost import sm_clock  # noqa: E402

SETTINGS = ("off_p0", "on_p0", "off_p20", "on_p20", "off_p50", "on_p50")
RUNS = (("pipeline_imix", "pipeline_up"), ("antispoof_64", "antispoof_ingress"))


def to_delegated(headers, share, seed, S):
    """A copy of the headers with about `share` of the frames turned into UDP over IPv6 from a random host in the
    delegated /56 (2001:db9:<s>::/56) of the subscriber whose IPv4 source the frame carried (a frame whose source is
    no subscriber's keeps a random subscriber's prefix: its MAC's binding does not own it)."""
    h = headers.copy()
    r = np.random.default_rng(seed)
    sub_of = {bytes(b): s for s, b in enumerate(S.ip_bytes(S.sub_ip(np.arange(N_SUBS))).reshape(-1, 4))}
    pick = np.nonzero(r.random(len(h)) < share)[0]
    s = np.array([sub_of.get(bytes(h[i, 26:30]), -1) for i in pick], np.int64)
    s = np.where(s >= 0, s, r.integers(0, N_SUBS, len(pick)))
    h[pick, 12], h[pick, 13], h[pick, 14], h[pick, 20], h[pick, 21] = 0x86, 0xDD, 0x60, 17, 64
    a = np.zeros((len(pick), 16), np.uint8)
    a[:, 0], a[:, 1], a[:, 2], a[:, 3] = 0x20, 0x01, 0x0D, 0xB9
    a[:, 4], a[:, 5] = s >> 8, s & 0xFF
    a[:, 7] = r.integers(0, 256, len(pick), dtype=np.uint8)  # any /64 of the /56
    a[:, 8:] = r.integers(0, 256, (len(pick), 8), dtype=np.uint8)
    h[pick, 22:38] = a
    return h


def workload_cost(name, prog, frames, steps, rounds):
    import torch
    from bng_b200 import layouts as L
    from bng_b200 import synth as S
    from bng_b200 import workloads as W
    dev = torch.device("cuda")
    rigs = {}
    for s in SETTINGS:
        wl = W.build(name, frames, 0, 1, 1)
        wl.prog = prog
        rigs[s] = Rig(wl, torch, dev)
    wl = rigs["off_p0"].wl
    if wl.derive is not None:
        wl.headers, wl.lens = wl.derive(rigs["off_p0"].translated)
    keys, owners = prefixes(S, L)
    for s, r in rigs.items():
        share = int(s.split("_p")[1]) / 100
        r.stage(to_delegated(wl.headers, share, 11, S) if share else wl.headers, wl.lens)
        assert r.dp.ipv6_prefixes_set(keys["addr"], keys["prefixlen"], owners) == 0
        if s.startswith("on"):
            r.dp.antispoof_ipv6_prefixes_enable(True)
    res = {"frames": wl.n, "prog": prog, "mpps": {s: [] for s in SETTINGS}, "dropped_per_batch": {},
           "launches_per_batch": {}}
    for s in SETTINGS:  # warm up every setting
        rigs[s].timed(2)
    for _ in range(rounds):
        for s in SETTINGS:
            mpps, _ = rigs[s].timed(steps)
            res["mpps"][s].append(round(mpps, 1))
    for s in SETTINGS:
        r = rigs[s]
        r.dp.prof_enable(True)
        n0 = r.dp.launch_count
        for _ in range(5):
            r.restore()
            r.step()
            r.dp.sync()
        res["launches_per_batch"][s] = (r.dp.launch_count - n0) // 5
        res["dropped_per_batch"][s] = int((r.verdict_d == L.TC_ACT_SHOT).sum().item())
        prof = r.dp.prof_read()
        r.dp.prof_enable(False)
        r.restore()
        res["kernels_ms_" + s] = {k: round(v[1] / v[0], 4) for k, v in prof.items() if "k_pipe_classify" in k or "k_antispoof" in k}
    for r in rigs.values():
        r.dp.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=1 << 22)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "workloads": {}}
    for name, prog in RUNS:
        res["workloads"][f"{name}/{prog}"] = workload_cost(name, prog, a.frames, a.steps, a.rounds)
    res["card"].update(sm_clock())
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
