"""What incremental replication costs: bng_delta_export time and blob size against bng_snapshot's, bng_delta_apply time on
a standby, and pipeline_imix Mpps with change tracking enabled and disabled, alternated on one context.

    python tools/delta_cost.py [--frames 4194304] [--steps 5] [--rounds 3] [--out FILE]

Exports are measured at the headline population (tables sized for the workload, as bench.py sizes them) and at the
reference's capacities (1 M subscribers, 4 M sessions, 2 M EIM mappings), for
  - steady traffic (nat_steady_64): one batch after the baseline, exported with refresh_ns = 1 s;
  - cold traffic (nat_cold_64): the first batch of new flows after the baseline.
Times are host wall clock around calls that end synchronised.  Prints one JSON document with the card and its power
limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
    if q:
        out["power_limit"], out["max_sm_clock"] = [x.strip() for x in q[0].split(",")]
    return out


def _ms(fn):
    t0 = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t0) * 1e3, r


def _load(dp, wl, dev):
    import torch
    from bng_b200 import MEM_DEVICE
    from bng_b200.layouts import as_bytes
    for m, k, v in wl.maps:
        assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
    for prog, h, l in wl.prewarm:
        ph, pl = torch.from_numpy(h).to(dev).reshape(-1), torch.from_numpy(l.astype(np.int32)).to(dev)
        torch.cuda.synchronize()
        dp.run(prog, ph, pl, wl.now0 - 1, stride=64, mem=MEM_DEVICE)
        dp.sync()


def _batch(dp, wl, dev, now):
    import torch
    from bng_b200 import MEM_DEVICE
    h = torch.from_numpy(wl.headers).to(dev).reshape(-1)
    l = torch.from_numpy(wl.lens.astype(np.int32)).to(dev)
    torch.cuda.synchronize()
    dp.run(wl.prog, h, l, now, stride=64, mem=MEM_DEVICE)
    dp.sync()
    for ring in ("spoof_events", "nat_log_rb"):
        dp.drain(ring)


def export_cost(name, frames, caps, dev):
    from bng_b200 import Dataplane
    from bng_b200 import layouts as L
    from bng_b200 import workloads as W
    wl = W.build(name, frames)
    opts = {} if caps == "reference" else W.sizing(wl)
    a, b = Dataplane(max_batch=frames, **opts), Dataplane(max_batch=frames, **opts)
    try:
        a.delta_enable()
        _load(a, wl, dev)
        cold = name == "nat_cold_64"
        if not cold:
            _batch(a, wl, dev, wl.now0)
        full_ms, full = _ms(lambda: a.delta_export(refresh_ns=10**9))
        apply_full_ms, _ = _ms(lambda: b.delta_apply(full))
        _batch(a, wl, dev, wl.now0 + wl.now_step)
        inc_ms, inc = _ms(lambda: a.delta_export(refresh_ns=10**9))
        apply_inc_ms, rc = _ms(lambda: b.delta_apply(inc))
        assert rc == 0
        idle_ms, idle = _ms(lambda: a.delta_export(refresh_ns=10**9))
        snap_ms, snap = _ms(a.snapshot)
        sec = L.parse_delta(inc)[1]["nat_sessions"]
        return {"workload": name, "capacities": caps, "sessions": int(a.map_info("nat_sessions")["count"]),
                "full_export_ms": round(full_ms, 2), "full_bytes": len(full), "full_apply_ms": round(apply_full_ms, 2),
                "export_ms": round(inc_ms, 2), "bytes": len(inc), "session_upserts": int(sec[2].shape[0]),
                "apply_ms": round(apply_inc_ms, 2), "unchanged_export_ms": round(idle_ms, 2), "unchanged_bytes": len(idle),
                "snapshot_ms": round(snap_ms, 2), "snapshot_bytes": len(snap)}
    finally:
        a.close()
        b.close()


def tracking_mpps(frames, steps, rounds, dev):
    """pipeline_imix, device-resident: Mpps per round with tracking off and on (the same context, toggled)."""
    import torch
    from bng_b200 import MEM_DEVICE, Dataplane
    from bng_b200 import workloads as W
    wl = W.build("pipeline_imix", frames)
    dp = Dataplane(max_batch=frames, **W.sizing(wl))
    try:
        _load(dp, wl, dev)
        hw = wl.headers.shape[1]
        off16, stride, total16 = W.slot16(wl.lens, wl.imix, hw, 64)
        hdr = torch.from_numpy(wl.headers).to(dev)
        arena = torch.zeros(total16 * 16 + 64, dtype=torch.uint8, device=dev)
        gidx = torch.from_numpy(off16.astype(np.int64)).to(dev)[:, None] + torch.arange(hw // 16, device=dev)[None, :]
        off_d = torch.from_numpy(off16.astype(np.int32)).to(dev)
        len0 = torch.from_numpy(wl.lens.astype(np.int32)).to(dev)
        lens, verdict = len0.clone(), torch.zeros(wl.n, dtype=torch.uint8, device=dev)
        stream = torch.cuda.ExternalStream(dp.stream, device=dev)
        out = {"off": [], "on": []}
        k = 0
        for r in range(rounds + 1):  # round 0 warms up
            for setting in ("off", "on"):
                dp.delta_enable(setting == "on")
                ms = 0.0
                for _ in range(steps):
                    arena[: total16 * 16].view(total16, 16)[gidx.reshape(-1)] = hdr.view(-1, 16)
                    lens.copy_(len0)
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    dp.run(wl.prog, arena, lens, wl.now0 + k * wl.now_step, off16=off_d, stride=0, verdict=verdict,
                           mem=MEM_DEVICE)
                    e1.record(stream)
                    dp.sync()
                    ms += e0.elapsed_time(e1)
                    k += 1
                    for ring in ("spoof_events", "nat_log_rb"):
                        dp.drain(ring)
                if r:
                    out[setting].append(round(wl.n * steps / (ms * 1e-3) / 1e6, 1))
        return out
    finally:
        dp.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1 << 22)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    dev = torch.device("cuda")
    res = {"card": card(), "frames": a.frames, "exports": []}
    for caps in ("headline", "reference"):
        for name in ("nat_steady_64", "nat_cold_64"):
            res["exports"].append(export_cost(name, a.frames, caps, dev))
    res["pipeline_imix_mpps"] = tracking_mpps(a.frames, a.steps, a.rounds, dev)
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
