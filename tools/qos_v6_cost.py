"""What shaping IPv6 frames with their owner's token bucket (bng_qos_ipv6_enable) costs the device-resident step:
pipeline_imix run as pipeline_up and as pipeline_tc, qos_64 (qos_ingress_prog) and qos_egress_64 (qos_egress_prog) at
2^22 frames, the settings alternated in one process over several rounds.  As in tools/dualstack_cost.py, every
subscriber's antispoof binding carries an IPv6 address inside its /64 and upstream IPv6 frames are sent from it, so
that they pass antispoof and are shaped:
    off       shaping off, the table empty (the kernels of a context that never used either)
    on_empty  shaping on, the table empty (must launch what "off" launches)
    on_p0     shaping on, 10 k subscribers x 2 prefixes (a /64 and a delegated /56), no IPv6 frames
    on_p20    the same, about 20 % of the frames turned into IPv6 frames of those subscribers' prefixes
    on_p50    the same, about 50 %

    python tools/qos_v6_cost.py [--steps 10] [--rounds 3] [--out FILE]

Prints one JSON document: the card (name, power limit, SM clock read after the runs), Mpps per round and setting,
and the classify / resolve kernel times of a profiled pass per setting (device events, bng_prof_*)."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from dualstack_cost import bind_ipv6, prefixes, to_ipv6  # noqa: E402
from li_cost import Rig, card  # noqa: E402

SETTINGS = ("off", "on_empty", "on_p0", "on_p20", "on_p50")
RUNS = (("pipeline_imix", "pipeline_up"), ("pipeline_imix", "pipeline_tc"), ("qos_64", "qos_ingress_prog"),
        ("qos_egress_64", "qos_egress_prog"))


def sm_clock():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm,power.limit,power.draw", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(("sm_clock", "max_sm_clock", "power_limit", "power_draw"), [x.strip() for x in q.split(",")]))
    except Exception as e:  # noqa: BLE001 - informational only
        return {"sm_clock": f"unknown ({e})"}


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
    wl = rigs["off"].wl
    if wl.derive is not None:
        wl.headers, wl.lens = wl.derive(rigs["off"].translated)
    keys, owners = prefixes(S, L)
    up = prog != "qos_egress_prog"
    src_of_mac = {}
    for r in rigs.values():  # the same bindings everywhere: IPv4 frames are unaffected by an IPv6 address
        src_of_mac = bind_ipv6(r.dp, S, L)
    for s, r in rigs.items():
        share = {"on_p20": 0.2, "on_p50": 0.5}.get(s, 0.0)
        r.stage(to_ipv6(wl.headers, share, up, 11, src_of_mac) if share else wl.headers, wl.lens)
        if s != "off":
            r.dp.qos_ipv6_enable(True)
        if s not in ("off", "on_empty"):
            assert r.dp.ipv6_prefixes_set(keys["addr"], keys["prefixlen"], owners) == 0
    res = {"frames": wl.n, "prog": prog, "ipv6_bound_macs": len(src_of_mac), "mpps": {s: [] for s in SETTINGS},
           "dropped_per_batch": {}, "launches_per_batch": {}}
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
        res["kernels_ms_" + s] = {k: round(v[1] / v[0], 4) for k, v in prof.items() if "classify" in k or "resolve" in k}
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
