"""What a NAT flow-state flush costs at the reference's capacities (4 M sessions, 2 M EIM mappings): bng_nat_flush of
1, 1 000 and 100 000 addresses, bng_sweep with nothing to expire, and the host alternative for one subscriber (dump
nat_sessions, delete the subscriber's keys one by one).  The tables are filled first with pipeline_imix's flows.

    python tools/flush_cost.py [--reps 10] [--out FILE]

Prints one JSON document: the card, its power limit and SM clock, and per measurement the device-event time of the
call on the context's stream, the host time of the call, the k_nat_flush / k_nat_sweep kernel time (bng_prof), and
what the call removed.  `pass_bytes` is the lower bound of the pass computed from the table sizes: one 32-byte sector
per slot of nat_sessions, nat_reverse and eim_table."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NS = 10**9


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        out["power_limit"], out["max_sm_clock"], out["sm_clock_now"] = [x.strip() for x in q.split(",")]
    except Exception as e:  # noqa: BLE001 - informational only
        out["power_limit"] = f"unknown ({e})"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from bng_b200 import Dataplane
    from bng_b200 import synth as S
    from bng_b200 import workloads as W
    from bng_b200.layouts import as_bytes
    if not torch.cuda.is_available():
        raise SystemExit("flush_cost.py measures on a CUDA device; none is present")
    dev = torch.device("cuda")
    res = {"card": card()}
    wl = W.build("pipeline_imix", 1 << 20)
    dp = Dataplane(max_batch=1 << 20)  # the reference's capacities
    for m, k, v in wl.maps:
        assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
    for prog, h, l in wl.prewarm:
        dp.run(prog, h.reshape(-1).copy(), l.copy(), wl.now0 - 1, stride=64)
    dp.drain("nat_log_rb")
    info = {m: dp.map_info(m) for m in ("nat_sessions", "nat_reverse", "eim_table", "subscriber_nat")}
    res["tables"] = {m: {"count": int(i["count"]), "max_entries": int(i["max_entries"])} for m, i in info.items()}
    slots = {"nat_sessions": 1 << 23, "nat_reverse": 1 << 23, "eim_table": 1 << 22}  # powers of two >= 2 x max_entries
    res["pass_bytes"] = sum(32 * s for s in slots.values())
    lib_stream = torch.cuda.ExternalStream(dp.stream, device=dev)
    subs = np.ascontiguousarray(dp.dump("subscriber_nat")[0]).view("<u4").reshape(-1)
    now = [wl.now0 + NS]

    def timed(call):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(lib_stream)
        t0 = time.perf_counter()
        out = call()
        t1 = time.perf_counter()
        e1.record(lib_stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), (t1 - t0) * 1e3, out

    def measure(name, make_call, kernel):
        for _ in range(3):  # warm-up
            make_call()()
        dp.prof_enable(True)
        ev, host, removed = [], [], []
        for _ in range(a.reps):
            e, h, out = timed(make_call())
            ev.append(e)
            host.append(h)
            removed.append(out)
        prof = dp.prof_read()
        dp.prof_enable(False)
        dp.drain("nat_log_rb")
        k = prof.get(kernel)
        r = {"event_ms_median": round(float(np.median(ev)), 4), "event_ms": [round(x, 4) for x in ev],
             "host_ms_median": round(float(np.median(host)), 4),
             "kernel_ms_mean": round(k[1] / k[0], 4) if k else None, "removed": removed}
        if k:
            r["pass_GBps"] = round(res["pass_bytes"] / (k[1] / k[0] * 1e-3) / 1e9, 1)
        res[name] = r

    cursor = [0]

    def flush_of(n):
        def make():
            # fresh subscribers while there are any, so that most timed calls remove state; then addresses without
            picks = np.arange(cursor[0], cursor[0] + n) % (2 * len(subs))
            cursor[0] += n
            addrs = np.where(picks < len(subs), subs[np.minimum(picks, len(subs) - 1)],
                             (0x0B000000 + picks).astype("<u4")).astype("<u4")
            now[0] += NS
            t = now[0]
            return lambda: list(dp.nat_flush(addrs, t))
        return make

    for n in (1, 1000, 100_000):
        measure(f"nat_flush_{n}", flush_of(n), "k_nat_flush")

    def sweep_call():
        now[0] += 1000  # nothing has been idle for 60 s
        t = now[0]
        return lambda: dp.sweep(t)

    measure("sweep_nothing_to_expire", sweep_call, "k_nat_sweep")

    # the host alternative for one subscriber: dump nat_sessions, then one synchronous delete per session
    dp.run(wl.prewarm[0][0], wl.prewarm[0][1].reshape(-1).copy(), wl.prewarm[0][2].copy(), now[0], stride=64)
    dp.drain("nat_log_rb")
    keys = dp.dump("nat_sessions")[0]
    src = np.ascontiguousarray(keys[:, :4]).view("<u4").reshape(-1)
    host = []
    for i in range(min(a.reps, 5)):
        sub = subs[i]
        t0 = time.perf_counter()
        k = dp.dump("nat_sessions")[0]
        mine = k[np.ascontiguousarray(k[:, :4]).view("<u4").reshape(-1) == sub]
        for row in mine:
            assert dp.delete("nat_sessions", row) == 0
        host.append({"ms": round((time.perf_counter() - t0) * 1e3, 2), "sessions": int(len(mine))})
    res["host_dump_and_delete_1"] = {"runs": host, "ms_median": float(np.median([h["ms"] for h in host])),
                                     "sessions_in_table": int(len(src))}
    res["card_after"] = card()
    dp.close()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
