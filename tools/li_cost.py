"""What lawful interception costs the device-resident step: pipeline_imix (pipeline_up, uplink) and nat_ingress_64
(nat44_ingress, downlink) at 2^22 frames, with interception never configured (one context), configured with no
target, and with 1, 100 and 1000 of the 10 k subscribers targeted (another context), alternated in one process.

    python tools/li_cost.py [--steps 10] [--rounds 3] [--out FILE]

Prints one JSON document: the card and its power limit, Mpps per round and setting, records per batch, and the
per-kernel times of a profiled pass at 1000 targets.  The ring is drained between steps, outside the timed region."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SETTINGS = ("never", "no_targets", "t1", "t100", "t1000")


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


class Rig:
    """One context with a workload's maps and prewarm, and the device arena of its timed batch."""

    def __init__(self, wl, torch, dev):
        from bng_b200 import MEM_DEVICE, Dataplane
        from bng_b200 import workloads as W
        from bng_b200.layouts import as_bytes
        self.torch, self.wl, n = torch, wl, wl.n
        self.dp = Dataplane(max_batch=max(n, 1 << 20), **W.sizing(wl))
        for m, k, v in wl.maps:
            assert self.dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
        translated = []
        for prog, h, l in wl.prewarm:
            ph = torch.from_numpy(h).to(dev).reshape(-1)
            pl = torch.from_numpy(l.astype(np.int32)).to(dev)
            torch.cuda.synchronize()
            self.dp.run(prog, ph, pl, wl.now0 - 1, stride=64, mem=MEM_DEVICE)
            self.dp.sync()
            translated.append(ph.cpu().numpy())
        self.translated = translated
        self.dev, self.MEM_DEVICE, self.step_no = dev, MEM_DEVICE, 0

    def stage(self, headers, lens):
        from bng_b200 import workloads as W
        torch, wl, dev = self.torch, self.wl, self.dev
        n, hw = wl.n, headers.shape[1]
        self.off16, self.stride, total16 = W.slot16(lens, wl.imix, hw, 64)
        self.hdr_d = torch.from_numpy(headers).to(dev)
        self.len0_d = torch.from_numpy(lens.astype(np.int32)).to(dev)
        self.len_d = self.len0_d.clone()
        self.arena_d = torch.zeros(total16 * 16 + 64, dtype=torch.uint8, device=dev)
        self.a16 = self.arena_d[: total16 * 16].view(total16, 16)
        self.off_d = self.gidx = None
        if self.off16 is not None:
            self.off_d = torch.from_numpy(self.off16.astype(np.int32)).to(dev)
            self.gidx = self.off_d.long()[:, None] + torch.arange(hw // 16, device=dev)[None, :]
        self.verdict_d = torch.zeros(n, dtype=torch.uint8, device=dev)
        self.stream = torch.cuda.ExternalStream(self.dp.stream, device=dev)
        self.drain_buf = None

    def restore(self):
        dp, n = self.dp, self.wl.n
        dp.sync()
        if self.off16 is None:
            self.arena_d[: n * self.stride].view(n, self.stride)[:, : self.hdr_d.shape[1]] = self.hdr_d
        else:
            self.a16[self.gidx.reshape(-1)] = self.hdr_d.view(-1, 16)
        self.len_d.copy_(self.len0_d)
        self.torch.cuda.synchronize()
        for ring in ("spoof_events", "nat_log_rb"):
            dp.drain(ring)
        return self.li_drain()

    def li_drain(self):
        rs = self.dp.li_record_size
        if not rs:
            return 0
        if self.drain_buf is None:
            self.drain_buf = np.zeros(self.li_cap * rs, np.uint8)
        got = ctypes.c_uint64(0)
        self.dp._chk(self.dp.lib.bng_li_drain(self.dp.h, self.drain_buf.ctypes.data, self.li_cap, ctypes.byref(got)), "li_drain")
        return got.value

    def step(self):
        wl = self.wl
        self.dp.run(wl.prog, self.arena_d, self.len_d, wl.now0 + self.step_no * wl.now_step, off16=self.off_d, stride=self.stride,
                    verdict=self.verdict_d, mem=self.MEM_DEVICE)
        self.step_no += 1

    def timed(self, k):
        torch = self.torch
        ms, recs = [], []
        for _ in range(k):
            recs.append(self.restore())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(self.stream)
            self.step()
            e1.record(self.stream)
            self.dp.sync()
            ms.append(e0.elapsed_time(e1))
        recs.append(self.restore())
        return self.wl.n * k / (sum(ms) * 1e-3) / 1e6, recs[1:]


def workload_cost(name, frames, steps, rounds):
    import torch
    from bng_b200 import synth as S
    from bng_b200 import workloads as W
    dev = torch.device("cuda")
    wl = W.build(name, frames, 0, 1, 1)
    rigs = {"never": Rig(wl, torch, dev), "li": Rig(W.build(name, frames, 0, 1, 1), torch, dev)}
    if wl.derive is not None:
        wl.headers, wl.lens = wl.derive(rigs["never"].translated)
    for r in rigs.values():
        r.stage(wl.headers, wl.lens)
        r.li_cap = 1 << 19
    rigs["li"].dp.li_configure(0, rigs["li"].li_cap)  # default snaplen (1518 bytes)
    targets = S.ip_bytes(S.sub_ip(np.arange(0, 10_000, 10))).view("<u4").reshape(-1)  # 1000 subscribers, spread out
    have = []

    def apply(setting):
        want = {"t1": 1, "t100": 100, "t1000": 1000}.get(setting, 0)
        dp = rigs["li"].dp
        while len(have) > want:
            assert dp.li_target_del(int(have.pop())) == 0
        while len(have) < want:
            a = int(targets[len(have)])
            dp.li_target_set(a, len(have))
            have.append(a)
        return rigs["never" if setting == "never" else "li"]

    res = {"frames": wl.n, "prog": wl.prog, "mpps": {s: [] for s in SETTINGS}, "records_per_batch": {}}
    for s in SETTINGS:  # warm up every setting
        apply(s).timed(2)
    for _ in range(rounds):
        for s in SETTINGS:
            mpps, recs = apply(s).timed(steps)
            res["mpps"][s].append(round(mpps, 1))
            res["records_per_batch"][s] = int(np.median(recs)) if recs else 0
    res["li_lost"] = rigs["li"].dp.li_lost
    res["launches_equal_never_vs_no_targets"] = None
    for s in ("never", "no_targets"):  # launches of one step
        r = apply(s)
        r.restore()
        c0 = r.dp.launch_count
        r.step()
        r.dp.sync()
        res.setdefault("launches_per_step", {})[s] = r.dp.launch_count - c0
    res["launches_equal_never_vs_no_targets"] = res["launches_per_step"]["never"] == res["launches_per_step"]["no_targets"]
    for s in ("no_targets", "t1000"):
        r = apply(s)
        r.dp.prof_enable(True)
        for _ in range(5):
            r.restore()
            r.step()
            r.dp.sync()
        prof = r.dp.prof_read()
        r.dp.prof_enable(False)
        r.restore()
        res["kernels_ms_" + s] = {k: round(v[1] / v[0], 4) for k, v in prof.items()}
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
    for name in ("pipeline_imix", "nat_ingress_64"):
        res["workloads"][name] = workload_cost(name, a.frames, a.steps, a.rounds)
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
