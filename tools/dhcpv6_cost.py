"""What the DHCPv6 fast path (bng_dhcpv6_enable) costs dhcp_fastpath_prog, on the GPU, settings alternated in one process
over several rounds:
    dhcp_off / dhcp_on   bench.py's DHCPv4 workload (`dhcp`, 2^22 frames, 384-byte slots) with the switch off and on
                         (on: a configured server and 1 M DHCPv6 bindings, so k_dhcp_fastpath<v6> runs)
    v6_384 / v6_512      2^22 DHCPv6 frames from 1 M bound clients, Solicit / Request / Renew / Rebind in equal parts,
                         in 384-byte slots (tile mode) and 512-byte slots (frame by frame)
Device-resident batches; the kernel time is from device events (bng_prof_*), Mpps from it.  Then whole calls on the
pinned zero-copy feed (BNG_MEM_HOST, host clock around the synchronised call) for v6_512.

    python tools/dhcpv6_cost.py [--rounds 3] [--steps 10] [--out FILE]

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
N_CLIENTS = 1 << 20
T0 = 1_000_000 * 1_000_000_000
SERVER_DUID = bytes.fromhex("000300010a0b0c0d0e0f")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def client_duid(i):
    return b"\x00\x01\x00\x01" + (0x2A000000 + i).to_bytes(4, "big") + (0x020000000000 + i).to_bytes(6, "big")


def v6_tables():
    cfg = np.zeros(1, L.bng_dhcpv6_server_config)
    cfg["server_mac"] = [[0x02, 0xAA, 0xBB, 0xCC, 0xDD, 0x01]]
    cfg["duid_len"], cfg["dns_count"] = len(SERVER_DUID), 2
    cfg["server_ip"][0] = np.frombuffer(bytes.fromhex("fe800000000000000000000000000001"), np.uint8)
    cfg["duid"][0, :10] = np.frombuffer(SERVER_DUID, np.uint8)
    cfg["dns"][0, 0, :2], cfg["dns"][0, 1, :2] = [0x20, 0x01], [0x20, 0x01]
    i = np.arange(N_CLIENTS, dtype=np.uint64)
    keys = np.zeros(N_CLIENTS, L.bng_dhcpv6_client_key)
    keys["duid_len"] = 14
    keys["duid"][:, :4] = [0, 1, 0, 1]
    keys["duid"][:, 4:8] = S.ip_bytes((np.uint64(0x2A000000) + i).astype(np.uint32))
    keys["duid"][:, 8:14] = S.mac_bytes(np.uint64(0x020000000000) + i)
    vals = np.zeros(N_CLIENTS, L.bng_dhcpv6_binding)
    vals["mac"] = S.mac_bytes(np.uint64(0x020000000000) + i)
    vals["flags"], vals["pd_len"], vals["iaid_na"], vals["iaid_pd"] = 3, 56, 1, 2
    vals["preferred_lft"], vals["valid_lft"], vals["expires_s"] = 3600, 7200, 1 << 40
    vals["addr"][:, 0], vals["prefix"][:, 0] = 0x20, 0x20
    return cfg, keys, vals


def v6_frames(stride, seed=5):
    """2^22 requests in `stride`-byte slots: four templates (client 0) patched with each frame's client."""
    tmpl = []
    for t in (1, 3, 5, 6):
        o = S.dhcpv6_option(1, client_duid(0))
        if t in (3, 5):
            o += S.dhcpv6_option(2, SERVER_DUID)
        o += S.dhcpv6_ia(3, 1) + S.dhcpv6_ia(25, 2) + S.dhcpv6_option(6, b"\x00\x17")
        tmpl.append(S.dhcpv6_frame(bytes.fromhex("020000000000"), t, 0x1234, o))
    rng = np.random.default_rng(seed)
    c = rng.integers(N_CLIENTS, size=N).astype(np.uint64)
    kind = rng.integers(4, size=N)
    a = np.zeros((N, stride), np.uint8)
    lens = np.zeros(N, np.uint32)
    for k, f in enumerate(tmpl):
        sel = kind == k
        a[sel, :len(f)] = np.frombuffer(f, np.uint8)
        lens[sel] = len(f)
    mac = S.mac_bytes(np.uint64(0x020000000000) + c)
    a[:, 6:12] = mac
    a[:, 70 + 4:70 + 8] = S.ip_bytes((np.uint64(0x2A000000) + c).astype(np.uint32))  # the Client ID's data at 70
    a[:, 70 + 8:70 + 14] = mac
    return a.reshape(-1), lens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda")
    dp = Dataplane(max_subscribers=N_CLIENTS, max_batch=N)
    wl = W.build("dhcp", N)
    for name, k, v in wl.maps:
        dp.update_batch(name, k, v)
    cfg, keys, vals = v6_tables()
    assert dp.update("dhcpv6_server_config", np.uint32(0), cfg) == 0
    for s in range(0, N_CLIENTS, 1 << 18):
        assert dp.update_batch("dhcpv6_bindings", keys[s:s + (1 << 18)], vals[s:s + (1 << 18)]) == 0
    hdr = wl.headers
    a4 = np.zeros((N, 384), np.uint8)
    a4[:, :hdr.shape[1]] = hdr
    sets = {"dhcp": (a4.reshape(-1), wl.lens, 384)}
    for stride in (384, 512):
        a, ln = v6_frames(stride)
        sets[f"v6_{stride}"] = (a, ln, stride)
    staged = {k: (torch.from_numpy(a).to(dev), torch.from_numpy(ln.view(np.int32)).to(dev), s) for k, (a, ln, s) in sets.items()}
    work = {k: (a.clone(), ln.clone(), s) for k, (a, ln, s) in staged.items()}
    verdict = torch.zeros(N, dtype=torch.uint8, device=dev)
    pid = dp.prog_id("dhcp_fastpath_prog")
    settings = [("dhcp_off", "dhcp", False), ("dhcp_on", "dhcp", True), ("v6_384", "v6_384", True), ("v6_512", "v6_512", True)]

    def one(setname, on, steps):
        dp.dhcpv6_enable(on)
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
        name = "k_dhcp_fastpath<v6>" if on else "k_dhcp_fastpath"
        n, ms = prof[name]
        return ms / n

    out = {"card": card(), "frames": N, "bindings": N_CLIENTS, "rounds": []}
    for _, s, on in settings:  # warm-up
        one(s, on, 2)
    for r in range(args.rounds):
        row = {}
        for label, s, on in settings:
            ms = one(s, on, args.steps)
            row[label] = {"ms": round(ms, 4), "Mpps": round(N / ms / 1e3, 1)}
        out["rounds"].append(row)
    st = dp.stats("dhcpv6_stats")
    out["dhcpv6_stats_last"] = dict(zip(L.DHCPV6_STATS, map(int, st)))
    # whole calls on the pinned zero-copy feed
    a, ln, stride = sets["v6_512"]
    pa = torch.from_numpy(a).pin_memory()
    pl = torch.from_numpy(ln.view(np.int32)).pin_memory()
    pv = torch.zeros(N, dtype=torch.uint8).pin_memory()
    calls = {}
    for on in (False, True, False, True):
        dp.dhcpv6_enable(on)
        ts = []
        for _ in range(args.steps):
            pa.copy_(torch.from_numpy(a))
            pl.copy_(torch.from_numpy(ln.view(np.int32)))
            t = time.perf_counter()
            dp.run(pid, pa, pl, T0, stride=stride, verdict=pv, mem=MEM_HOST, arena_bytes=a.nbytes)
            ts.append((time.perf_counter() - t) * 1e3)
        calls.setdefault("on" if on else "off", []).append(round(float(np.median(ts)), 3))
    out["pinned_v6_512_ms_per_call"] = calls
    out["card_after"] = card()
    js = json.dumps(out, indent=1)
    print(js)
    if args.out:
        with open(args.out, "w") as f:
            f.write(js)
    dp.close()


if __name__ == "__main__":
    main()
