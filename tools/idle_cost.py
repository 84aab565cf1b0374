"""What per-subscriber idle detection costs: pipeline_imix (pipeline_up) with accounting alone against accounting plus
idle detection, and with nothing against idle detection alone, alternated in one process on one context; plus the
time of bng_idle_scan at 10^6 subscribers (the default capacities) with 0 %, 1 % and 100 % of them idle.

    python tools/idle_cost.py [--steps 20] [--rounds 3] [--out FILE]

Prints one JSON document: the card and its power limit, Mpps per round and setting, the per-kernel times of a profiled
pass per setting, and the scan times (wall time of the call, and the k_idle_scan kernel alone)."""
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
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"] = [x.strip() for x in q.split(",")]
    except Exception as e:  # noqa: BLE001 - informational only
        out["power_limit"] = f"unknown ({e})"
    return out


SETTINGS = {"none": (False, False), "acct": (True, False), "idle": (False, True), "acct+idle": (True, True)}


def workload_cost(name, frames, steps, rounds, pairs):
    import torch
    from bng_b200 import MEM_DEVICE, Dataplane
    from bng_b200 import workloads as W
    from bng_b200.layouts import as_bytes
    dev = torch.device("cuda")
    wl = W.build(name, frames, 0, 1, 1)
    n = wl.n
    dp = Dataplane(max_batch=max(n, 1 << 20), **W.sizing(wl))
    for m, k, v in wl.maps:
        assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
    translated = []
    for prog, h, l in wl.prewarm:
        ph = torch.from_numpy(h).to(dev).reshape(-1)
        pl = torch.from_numpy(l.astype(np.int32)).to(dev)
        torch.cuda.synchronize()
        dp.run(prog, ph, pl, wl.now0 - 1, stride=64, mem=MEM_DEVICE)
        dp.sync()
        translated.append(ph.cpu().numpy())
    if wl.derive is not None:
        wl.headers, wl.lens = wl.derive(translated)
    hw = wl.headers.shape[1]
    off16, stride, total16 = W.slot16(wl.lens, wl.imix, hw, 64)
    hdr_d = torch.from_numpy(wl.headers).to(dev)
    len0_d = torch.from_numpy(wl.lens.astype(np.int32)).to(dev)
    len_d = len0_d.clone()
    arena_d = torch.zeros(total16 * 16 + 64, dtype=torch.uint8, device=dev)
    a16 = arena_d[: total16 * 16].view(total16, 16)
    off_d = gidx = None
    if off16 is not None:
        off_d = torch.from_numpy(off16.astype(np.int32)).to(dev)
        gidx = off_d.long()[:, None] + torch.arange(hw // 16, device=dev)[None, :]
    verdict_d = torch.zeros(n, dtype=torch.uint8, device=dev)
    lib_stream = torch.cuda.ExternalStream(dp.stream, device=dev)
    step_no = [0]

    def restore():
        dp.sync()
        if off16 is None:
            arena_d[: n * stride].view(n, stride)[:, :hw] = hdr_d
        else:
            a16[gidx.reshape(-1)] = hdr_d.view(-1, 16)
        len_d.copy_(len0_d)
        torch.cuda.synchronize()
        for ring in ("spoof_events", "nat_log_rb"):
            dp.drain(ring)

    def step():
        dp.run(wl.prog, arena_d, len_d, wl.now0 + step_no[0] * wl.now_step, off16=off_d, stride=stride, verdict=verdict_d,
               mem=MEM_DEVICE)
        step_no[0] += 1

    def timed(k):
        evs = []
        for _ in range(k):
            restore()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(lib_stream)
            step()
            e1.record(lib_stream)
            evs.append((e0, e1))
        dp.sync()
        torch.cuda.synchronize()
        return n * k / (sum(a.elapsed_time(b) for a, b in evs) * 1e-3) / 1e6

    def setting(s):
        acct, idle = SETTINGS[s]
        dp.acct_enable(wl.prog, acct)
        dp.idle_enable(wl.prog, idle)

    res = {"frames": n, "prog": wl.prog}
    for pair in pairs:
        mp = {s: [] for s in pair}
        for s in pair:  # warm up both settings
            setting(s)
            timed(3)
        for _ in range(rounds):
            for s in pair:
                setting(s)
                mp[s].append(round(timed(steps), 1))
        res[" vs ".join(pair)] = mp
    for s in SETTINGS:
        setting(s)
        dp.prof_enable(True)
        for _ in range(5):
            restore()
            step()
            dp.sync()
        prof = dp.prof_read()
        dp.prof_enable(False)
        res["kernels_ms_" + s] = {k: round(v[1] / v[0], 4) for k, v in prof.items()}
    dp.close()
    return res


def scan_cost(n=1_000_000, reps=5):
    import ctypes
    from bng_b200 import Dataplane, synth as S
    from bng_b200.layouts import IDLE_NEVER, bng_idle, token_bucket
    out = {}
    dp = Dataplane(max_batch=1 << 16)  # the default capacities: 10^6 subscribers, 2^21 directory slots
    keys = S.ip_bytes(S.sub_ip(np.arange(n)))
    assert dp.update_batch("qos_ingress", keys, np.zeros(n, token_bucket)) == 0
    dp.idle_enable("qos_ingress_prog")
    t0 = 10**12
    assert dp.lib.bng_idle_scan(dp.h, t0, 0, 3, None, None, 0) == 0  # starts every record
    addrs = np.zeros(n, "<u4")
    recs = np.zeros(n, bng_idle)
    rng = np.random.Generator(np.random.PCG64(1))
    for pct in (0, 1, 100):
        tos = np.full(n, IDLE_NEVER, np.uint32)
        tos[rng.random(n) < pct / 100] = 1
        assert dp.idle_timeout_set(keys, tos).all()
        want = int((tos == 1).sum())
        ts = []
        dp.prof_enable(True)
        for _ in range(reps):
            t = time.perf_counter()
            got = dp.lib.bng_idle_scan(dp.h, t0 + 5 * 10**9, 0, 3, addrs.ctypes.data, recs.ctypes.data, ctypes.c_uint64(n))
            ts.append((time.perf_counter() - t) * 1e3)
            assert got == want, (got, want)
        prof = dp.prof_read()
        dp.prof_enable(False)
        k = prof.get("k_idle_scan", (1, 0.0))
        out[f"{pct}%"] = {"idle": want, "ms_median": round(float(np.median(ts)), 3), "ms": [round(x, 3) for x in ts],
                          "k_idle_scan_ms": round(k[1] / k[0], 4)}
    dp.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=1 << 22)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    res["pipeline_imix"] = workload_cost("pipeline_imix", a.frames, a.steps, a.rounds, [("acct", "acct+idle"), ("none", "idle")])
    res["idle_scan_1M"] = scan_cost()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
