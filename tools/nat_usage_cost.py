"""What the NAT port-usage census (bng_nat_usage) costs: the wall time of the call and the times of its kernels at the
pipeline_imix state (10 k subscribers) and at the reference's full capacities (nat_cold_64 with 2^22 new flows), and
pipeline_imix Mpps with and without a census every N batches, alternated in one process on one context.

    python tools/nat_usage_cost.py [--steps 20] [--rounds 3] [--every 8] [--out FILE]

Prints one JSON document with the card and its power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from idle_cost import card  # noqa: E402


def census_cost(dp, reps=7):
    """Median wall time of bng_nat_usage (every record copied out) and its kernels' mean times."""
    dp.nat_usage()  # scratch allocated, shapes warmed
    ts = []
    for _ in range(reps):  # the wall time, profiling off
        t = time.perf_counter()
        s = dp.nat_usage()[0]
        ts.append((time.perf_counter() - t) * 1e3)
    dp.prof_enable(True)
    for _ in range(reps):
        dp.nat_usage()
    prof = dp.prof_read()
    dp.prof_enable(False)
    return {"summary": s, "ms_median": round(float(np.median(ts)), 3), "ms": [round(x, 3) for x in ts],
            "kernels_ms": {k: round(v[1] / v[0], 4) for k, v in prof.items() if k.startswith("k_natuse")}}


def pipeline_cost(frames, steps, rounds, every):
    import torch
    from bng_b200 import MEM_DEVICE, Dataplane
    from bng_b200 import workloads as W
    from bng_b200.layouts import as_bytes
    dev = torch.device("cuda")
    wl = W.build("pipeline_imix", frames, 0, 1, 1)
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

    def timed(k, census):
        """Mpps over k batches, each timed from its launch to the end of its run (or of the census that follows every
        `every`-th batch), by the host clock around a synchronised stream."""
        total = 0.0
        for i in range(k):
            restore()
            t = time.perf_counter()
            dp.run(wl.prog, arena_d, len_d, wl.now0 + step_no[0] * wl.now_step, off16=off_d, stride=stride, verdict=verdict_d,
                   mem=MEM_DEVICE)
            step_no[0] += 1
            if census and i % every == every - 1:
                dp.nat_usage(800)
            dp.sync()
            total += time.perf_counter() - t
        return n * k / total / 1e6

    restore()
    res = {"frames": n, "prog": wl.prog, "census_every": every, "census": census_cost(dp)}
    for c in (False, True):
        timed(3, c)
    mp = {"without": [], "with": []}
    for _ in range(rounds):
        for c in (False, True):
            mp["with" if c else "without"].append(round(timed(steps, c), 1))
    res["mpps"] = mp
    dp.close()
    return res


def full_capacity_cost(frames):
    from bng_b200 import Dataplane
    from bng_b200 import workloads as W
    from bng_b200.layouts import as_bytes
    wl = W.build("nat_cold_64", frames, subs_scale=4)
    dp = Dataplane(max_batch=wl.n)  # the reference's capacities: 1e6 subscribers, 4e6 sessions, 2e6 EIM mappings
    for m, k, v in wl.maps:
        assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
    dp.run(wl.prog, wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0, stride=64)
    res = {"frames": wl.n, "census": census_cost(dp)}
    dp.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--every", type=int, default=8)
    ap.add_argument("--frames", type=int, default=1 << 22)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    res["pipeline_imix"] = pipeline_cost(a.frames, a.steps, a.rounds, a.every)
    res["full_capacity"] = full_capacity_cost(a.frames)
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
