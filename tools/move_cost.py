"""What a subscriber hand-over costs at the reference's capacities (4 M sessions, 2 M EIM mappings, 1 M subscribers per
context): bng_sub_export read-only, bng_sub_export with BNG_SUB_DETACH, and bng_sub_import into a second context, for
1, 1 000 and 100 000 addresses (with their MACs).  The source's tables are filled first with pipeline_imix's flows;
pipeline_imix has 10 000 subscribers, so a set of 100 000 addresses is those 10 000 and 90 000 without state.

    python tools/move_cost.py [--reps 5] [--out FILE]

Prints one JSON document: the card, its power limit and SM clock, and per measurement the device-event time of the
call on the context's stream, the host time of the call, the kernel times of the call (bng_prof: k_move_select,
k_delta_emit, k_move_detach, the table-op and record kernels), and the blob size.  `pass_bytes` is the lower bound of
the export's pass computed from the table sizes: one 32-byte sector per slot of nat_sessions, nat_reverse and
eim_table.  After each timed detach and import the subscribers are moved back, untimed, so every repetition moves the
same state."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
NS = 10**9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from flush_cost import card
    from bng_b200 import Dataplane
    from bng_b200 import synth as S
    from bng_b200 import workloads as W
    from bng_b200.layouts import as_bytes
    if not torch.cuda.is_available():
        raise SystemExit("move_cost.py measures on a CUDA device; none is present")
    dev = torch.device("cuda")
    res = {"card": card()}
    wl = W.build("pipeline_imix", 1 << 20)
    src = Dataplane(max_batch=1 << 20)  # the reference's capacities
    dst = Dataplane(max_batch=1 << 16)
    for m, k, v in wl.maps:
        assert src.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
    for prog, h, l in wl.prewarm:
        src.run(prog, h.reshape(-1).copy(), l.copy(), wl.now0 - 1, stride=64)
    src.run(wl.prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0, stride=64)
    src.drain("nat_log_rb")
    info = {m: src.map_info(m) for m in ("nat_sessions", "nat_reverse", "eim_table", "subscriber_nat")}
    res["tables"] = {m: {"count": int(i["count"]), "max_entries": int(i["max_entries"])} for m, i in info.items()}
    slots = {"nat_sessions": 1 << 23, "nat_reverse": 1 << 23, "eim_table": 1 << 22}  # powers of two >= 2 x max_entries
    res["pass_bytes"] = sum(32 * s for s in slots.values())
    subs = np.ascontiguousarray(src.dump("subscriber_nat")[0]).view("<u4").reshape(-1)
    # subscriber i of the workload: address S.sub_ip(i), MAC S.sub_mac_key(i)
    n_subs = len(subs)
    all_ips = np.ascontiguousarray(S.ip_bytes(S.sub_ip(np.arange(n_subs)))).view("<u4").reshape(-1)
    all_macs = S.sub_mac_key(np.arange(n_subs))

    def timed(dp, call):
        stream = torch.cuda.ExternalStream(dp.stream, device=dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        t0 = time.perf_counter()
        out = call()
        t1 = time.perf_counter()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), (t1 - t0) * 1e3, out

    import ctypes as C

    def export(dp, addrs, macs, flags, room):
        # the C call with a buffer of the right size (the binding sizes its buffer by -ENOSPC, which would run it twice)
        buf = np.empty(room, np.uint8)
        n = C.c_uint64(0)
        r = dp.lib.bng_sub_export(dp.h, addrs.ctypes.data, len(addrs), macs.ctypes.data, len(macs), flags, buf.ctypes.data,
                                  room, C.byref(n))
        assert r == 0, r
        return buf[: n.value].tobytes()

    def summary(ev, host, prof, blob_bytes, extra=None):
        r = {"event_ms_median": round(float(np.median(ev)), 4), "event_ms": [round(x, 4) for x in ev],
             "host_ms_median": round(float(np.median(host)), 4),
             "kernels_ms_mean": {k: round(v[1] / v[0], 4) for k, v in prof.items()},
             "blob_bytes": blob_bytes}
        sel = prof.get("k_move_select")
        if sel:
            r["pass_GBps"] = round(res["pass_bytes"] / (sel[1] / sel[0] * 1e-3) / 1e9, 1)
        r.update(extra or {})
        return r

    for n in (1, 1000, 100_000):
        k = min(n, n_subs)
        pick = np.arange(0, n_subs, max(1, n_subs // k))[:k]
        addrs = np.ascontiguousarray(np.concatenate([all_ips[pick], (0x0B000000 + np.arange(n - k)).astype("<u4")]))
        macs = np.ascontiguousarray(all_macs[pick])
        blob = src.sub_export(addrs, macs)
        for _ in range(2):  # warm-up
            export(src, addrs, macs, 0, len(blob))
        src.prof_enable(True)
        ev, host = [], []
        for _ in range(a.reps):
            e, h, _ = timed(src, lambda: export(src, addrs, macs, 0, len(blob)))
            ev.append(e)
            host.append(h)
        prof = src.prof_read()
        src.prof_enable(False)
        res[f"export_{n}"] = summary(ev, host, prof, len(blob), {"subscribers_with_state": int(k)})
        det = {"ev": [], "host": []}
        imp = {"ev": [], "host": []}
        prof_d, prof_i = {}, {}
        for rep in range(a.reps + 1):  # the first repetition warms up
            src.prof_enable(rep > 0)
            e, h, b = timed(src, lambda: export(src, addrs, macs, 1, len(blob)))
            if rep:
                det["ev"].append(e), det["host"].append(h)
                for kk, v in src.prof_read().items():
                    p = prof_d.setdefault(kk, [0, 0.0])
                    p[0] += v[0]
                    p[1] += v[1]
            src.prof_enable(False)
            dst.prof_enable(rep > 0)
            e, h, _ = timed(dst, lambda: dst.sub_import(b))
            if rep:
                imp["ev"].append(e), imp["host"].append(h)
                for kk, v in dst.prof_read().items():
                    p = prof_i.setdefault(kk, [0, 0.0])
                    p[0] += v[0]
                    p[1] += v[1]
            dst.prof_enable(False)
            back = dst.sub_export(addrs, macs, detach=True)  # untimed: the state goes home
            assert src.sub_import(back) == 0
        res[f"export_detach_{n}"] = summary(det["ev"], det["host"], prof_d, len(b))
        res[f"import_{n}"] = summary(imp["ev"], imp["host"], prof_i, len(b))
    res["tables_after"] = {m: int(src.map_info(m)["count"]) for m in info}
    res["card_after"] = card()
    src.close()
    dst.close()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
