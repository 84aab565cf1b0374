"""What answering Router and Neighbor Solicitations (bng_nd_enable) costs dhcp_fastpath_prog, on the GPU, settings
alternated in one process over several rounds:
    dhcp_off / dhcp_on   bench.py's DHCPv4 workload (`dhcp`, 2^22 frames, 384-byte slots) with the switch off and on
                         (on: a configured nd_config and 1 M nd_bindings, so k_dhcp_fastpath<nd> runs)
    nd_384 / nd_512      2^22 ICMPv6 frames from 1 M bound subscribers, Router Solicitations and Neighbor Solicitations
                         for the router's link-local address in equal parts, in 384-byte slots (tile mode) and
                         512-byte slots (frame by frame); the RA carries two shared prefixes, the subscriber's own
                         prefix, two DNS servers and two search domains (262 bytes with its headers)
Device-resident batches; the kernel time is from device events (bng_prof_*), Mpps from it.  Then whole calls on the
pinned zero-copy feed (BNG_MEM_HOST, host clock around the synchronised call) for nd_512.

    python tools/nd_cost.py [--rounds 3] [--steps 10] [--out FILE]

Prints one JSON document with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bng_b200 import MEM_DEVICE, MEM_HOST, Dataplane  # noqa: E402
from bng_b200 import layouts as L  # noqa: E402
from bng_b200 import synth as S  # noqa: E402
from bng_b200 import workloads as W  # noqa: E402

N = 1 << 22
N_SUBS = 1 << 20
T0 = 1_000_000 * 1_000_000_000
ROUTER_MAC = bytes.fromhex("02aabbccdd01")
ROUTER_LL = bytes.fromhex("fe800000000000000000000000000001")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def nd_tables():
    """nd_config as pkg/slaac's buildRA lays it out (MTU 1500, two shared /64s, two DNS servers, two search domains),
    and 1 M bindings, a /64 each."""
    head = bytes([134, 0, 0, 0, 64, 0, 0x07, 0x08]) + bytes(8) + b"\x01\x01" + ROUTER_MAC + bytes([5, 1, 0, 0, 0, 0, 5, 0xDC])
    for p in (b"\x20\x01\x0d\xb8\xff", b"\x20\x01\x0d\xb8\xfe"):
        head += bytes([3, 4, 64, 0xC0, 0, 0x27, 0x8D, 0, 0, 0x09, 0x3A, 0x80]) + bytes(4) + p + bytes(11)
    tail = bytes([25, 5, 0, 0, 0, 0, 0x15, 0x18]) + (b"\x20\x01\x0d\xb8" + bytes(11) + b"\x53") * 2
    names = b"\x03isp\x07example\x00\x07example\x03net\x00"
    names += bytes((8 - (8 + len(names)) % 8) % 8)
    tail += bytes([31, (8 + len(names)) // 8, 0, 0, 0, 0, 0x15, 0x18]) + names
    cfg = np.zeros(1, L.bng_nd_config)
    cfg["router_mac"][0] = np.frombuffer(ROUTER_MAC, np.uint8)
    cfg["router_ll"][0] = np.frombuffer(ROUTER_LL, np.uint8)
    cfg["ra_head_len"], cfg["ra_tail_len"] = len(head), len(tail)
    cfg["ra"][0, :len(head) + len(tail)] = np.frombuffer(head + tail, np.uint8)
    i = np.arange(N_SUBS, dtype=np.uint64)
    keys = np.uint64(0x020000000000) + i
    vals = np.zeros(N_SUBS, L.bng_nd_binding)
    vals["prefix"][:, :4] = [0x20, 0x01, 0x0d, 0xb8]
    vals["prefix"][:, 4:8] = S.ip_bytes(i.astype(np.uint32))
    vals["prefix_len"], vals["pio_flags"] = 64, 0xC0
    vals["valid_lft"], vals["preferred_lft"], vals["expires_s"] = 7200, 3600, 1 << 40
    return cfg, keys, vals


def nd_frames(stride, seed=5):
    """2^22 solicitations in `stride`-byte slots: an RS and an NS (subscriber 0) patched with each frame's MAC and
    link-local source, their ICMPv6 checksums recomputed."""
    mac0 = bytes.fromhex("020000000000")
    tmpl = [S.rs_frame(mac0), S.ns_frame(mac0, ROUTER_LL)]
    rng = np.random.default_rng(seed)
    c = rng.integers(N_SUBS, size=N).astype(np.uint64)
    kind = rng.integers(2, size=N)
    a = np.zeros((N, stride), np.uint8)
    lens = np.zeros(N, np.uint32)
    mac = S.mac_bytes(np.uint64(0x020000000000) + c)
    for k, f in enumerate(tmpl):
        sel = np.nonzero(kind == k)[0]
        a[sel, :len(f)] = np.frombuffer(f, np.uint8)
        lens[sel] = len(f)
        rows = a[sel]
        rows[:, 6:12] = mac[sel]
        rows[:, 30], rows[:, 31:33] = mac[sel, 0] ^ 2, mac[sel, 1:3]  # the EUI-64 source address
        rows[:, 35:38] = mac[sel, 3:6]
        slla = 64 if k == 0 else 80  # the Source Link-Layer Address option's data: after the RS body, the NS target
        rows[:, slla:slla + 6] = mac[sel]
        rows[:, 56:58] = 0
        plen = len(f) - 54
        w = rows[:, 22:54 + plen].astype(np.uint32)
        s = (w[:, 0::2] << 8).sum(1) + w[:, 1::2].sum(1) + plen + 58
        while (s >> 16).any():
            s = (s & 0xFFFF) + (s >> 16)
        ck = ~s & 0xFFFF
        rows[:, 56], rows[:, 57] = ck >> 8, ck & 0xFF
        a[sel] = rows
    return a.reshape(-1), lens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda")
    dp = Dataplane(max_subscribers=N_SUBS, max_batch=N)
    wl = W.build("dhcp", N)
    for name, k, v in wl.maps:
        dp.update_batch(name, k, v)
    cfg, keys, vals = nd_tables()
    assert dp.update("nd_config", np.uint32(0), cfg) == 0
    for s in range(0, N_SUBS, 1 << 18):
        assert dp.update_batch("nd_bindings", keys[s:s + (1 << 18)], vals[s:s + (1 << 18)]) == 0
    hdr = wl.headers
    a4 = np.zeros((N, 384), np.uint8)
    a4[:, :hdr.shape[1]] = hdr
    sets = {"dhcp": (a4.reshape(-1), wl.lens, 384)}
    for stride in (384, 512):
        a, ln = nd_frames(stride)
        sets[f"nd_{stride}"] = (a, ln, stride)
    staged = {k: (torch.from_numpy(a).to(dev), torch.from_numpy(ln.view(np.int32)).to(dev), s) for k, (a, ln, s) in sets.items()}
    work = {k: (a.clone(), ln.clone(), s) for k, (a, ln, s) in staged.items()}
    verdict = torch.zeros(N, dtype=torch.uint8, device=dev)
    pid = dp.prog_id("dhcp_fastpath_prog")
    settings = [("dhcp_off", "dhcp", False), ("dhcp_on", "dhcp", True), ("nd_384", "nd_384", True), ("nd_512", "nd_512", True)]

    def one(setname, on, steps):
        dp.nd_enable(on)
        a0, l0, stride = staged[setname]
        a, ln, _ = work[setname]
        dp.prof_enable(True)
        torch.cuda.synchronize()
        with torch.cuda.stream(torch.cuda.ExternalStream(dp.stream, device=dev)):
            for _ in range(steps):
                a.copy_(a0)
                ln.copy_(l0)
                dp.run(pid, a, ln, T0, stride=stride, verdict=verdict, mem=MEM_DEVICE, arena_bytes=a.numel())
        dp.sync()
        prof = dp.prof_read()
        dp.prof_enable(False)
        n, ms = prof["k_dhcp_fastpath<nd>" if on else "k_dhcp_fastpath"]
        return ms / n, verdict

    out = {"card": card(), "frames": N, "bindings": N_SUBS, "rounds": []}
    for _, s, on in settings:  # warm-up
        one(s, on, 2)
    for r in range(args.rounds):
        row = {}
        for label, s, on in settings:
            ms, v = one(s, on, args.steps)
            row[label] = {"ms": round(ms, 4), "Mpps": round(N / ms / 1e3, 1)}
            if label.startswith("nd"):
                row[label]["answered"] = int((v == 3).sum().item())
        out["rounds"].append(row)
    st = dp.stats("nd_stats")
    out["nd_stats_total"] = dict(zip(L.ND_STATS, map(int, st)))
    # whole calls on the pinned zero-copy feed
    a, ln, stride = sets["nd_512"]
    pa = torch.from_numpy(a).pin_memory()
    pl = torch.from_numpy(ln.view(np.int32)).pin_memory()
    pv = torch.zeros(N, dtype=torch.uint8).pin_memory()
    calls = {}
    for on in (False, True, False, True):
        dp.nd_enable(on)
        ts = []
        for _ in range(args.steps):
            pa.copy_(torch.from_numpy(a))
            pl.copy_(torch.from_numpy(ln.view(np.int32)))
            t = time.perf_counter()
            dp.run(pid, pa, pl, T0, stride=stride, verdict=pv, mem=MEM_HOST, arena_bytes=a.nbytes)
            ts.append((time.perf_counter() - t) * 1e3)
        calls.setdefault("on" if on else "off", []).append(round(float(np.median(ts)), 3))
    out["pinned_nd_512_ms_per_call"] = calls
    out["card_after"] = card()
    js = json.dumps(out, indent=1)
    print(js)
    if args.out:
        with open(args.out, "w") as f:
            f.write(js)
    dp.close()


if __name__ == "__main__":
    main()
