"""What IPv6 attribution (subscriber_ipv6) costs the device-resident step: pipeline_imix (pipeline_up, uplink) and
nat_ingress_64 (nat44_ingress, downlink) at 2^22 frames, with accounting on and one interception target, alternated
in one process over several rounds.  Every subscriber's antispoof binding carries an IPv6 address inside its /64,
and upstream IPv6 frames are sent from it, so that they pass antispoof and are attributed:
    empty    the table empty (the kernels of a context that never used it)
    p0       10 k subscribers x 2 prefixes (a /64 and a delegated /56), no IPv6 frames
    p20      the same, about 20 % of the frames turned into IPv6 frames of those subscribers' prefixes
    p50      the same, about 50 %

    python tools/dualstack_cost.py [--steps 10] [--rounds 3] [--out FILE]

Prints one JSON document: the card and its power limit, Mpps per round and setting, and the k_acct / k_li_capture
times of a profiled pass per setting."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from li_cost import Rig, card  # noqa: E402

SETTINGS = ("empty", "p0", "p20", "p50")
N_SUBS = 10_000


def prefixes(S, L):
    """(keys, owners) of two prefixes per subscriber: 2001:db8:<s>::/64 and 2001:db9:<s>::/56 (s in 16 bits)."""
    s = np.arange(N_SUBS)
    keys = np.zeros(2 * N_SUBS, L.bng_ipv6_prefix_key)
    for j, (b, pl) in enumerate(((0xB8, 64), (0xB9, 56))):
        k = keys[j * N_SUBS:(j + 1) * N_SUBS]
        k["prefixlen"] = pl
        a = np.zeros((N_SUBS, 16), np.uint8)
        a[:, 0], a[:, 1], a[:, 2], a[:, 3] = 0x20, 0x01, 0x0D, b
        a[:, 4], a[:, 5] = s >> 8, s & 0xFF
        k["addr"] = a
    owners = np.tile(S.ip_bytes(S.sub_ip(s)).view("<u4").reshape(-1), 2)
    return keys, owners


def bind_ipv6(dp, S, L):
    """Gives every subscriber_bindings entry of a workload subscriber an IPv6 address, 2001:db8:<s>::1 (inside its
    /64), so that antispoof passes upstream IPv6 frames from it.  Returns {MAC key: that address}."""
    keys, vals = dp.dump("subscriber_bindings")
    if not len(keys):  # a downstream workload binds nobody
        return {}
    sub_of = {bytes(b): s for s, b in enumerate(S.ip_bytes(S.sub_ip(np.arange(N_SUBS))).reshape(-1, 4))}
    b = vals.copy().view(L.subscriber_binding).reshape(-1)
    out = {}
    for i in range(len(b)):
        s = sub_of.get(bytes(b[i]["ipv4_addr"]))
        if s is None:
            continue
        a = np.zeros(16, np.uint8)
        a[0], a[1], a[2], a[3], a[4], a[5], a[15] = 0x20, 0x01, 0x0D, 0xB8, s >> 8, s & 0xFF, 1
        b[i]["ipv6_addr"], b[i]["ipv6_valid"] = a, 1
        out[int(keys[i].view("<u8")[0])] = a
    assert dp.update_batch("subscriber_bindings", keys, b) == 0
    return out


def to_ipv6(headers, share, up, seed, src_of_mac):
    """A copy of the headers with about `share` of the frames turned into UDP over IPv6 from / to a subscriber's
    prefix (the address where the program's direction looks for it).  Upstream, a frame from a bound MAC carries the
    binding's IPv6 source, so that antispoof passes it and it is attributed."""
    h = headers.copy()
    r = np.random.default_rng(seed)
    pick = np.nonzero(r.random(len(h)) < share)[0]
    s = r.integers(0, N_SUBS, len(pick))
    h[pick, 12], h[pick, 13], h[pick, 14], h[pick, 20], h[pick, 21] = 0x86, 0xDD, 0x60, 17, 64
    off = 22 if up else 38
    a = np.zeros((len(pick), 16), np.uint8)
    a[:, 0], a[:, 1], a[:, 2] = 0x20, 0x01, 0x0D
    a[:, 3] = np.where(r.random(len(pick)) < 0.5, 0xB8, 0xB9)
    a[:, 4], a[:, 5] = s >> 8, s & 0xFF
    a[:, 8:] = r.integers(0, 256, (len(pick), 8), dtype=np.uint8)
    if up:
        mac = np.zeros(len(pick), np.uint64)
        for j in range(6):
            mac = (mac << np.uint64(8)) | h[pick, 6 + j].astype(np.uint64)
        for i, m in enumerate(mac.tolist()):
            if m in src_of_mac:
                a[i] = src_of_mac[m]
    h[pick, off:off + 16] = a
    return h


def workload_cost(name, frames, steps, rounds):
    import torch
    from bng_b200 import layouts as L
    from bng_b200 import synth as S
    from bng_b200 import workloads as W
    dev = torch.device("cuda")
    rigs = {s: Rig(W.build(name, frames, 0, 1, 1), torch, dev) for s in SETTINGS}
    wl = rigs["empty"].wl
    if wl.derive is not None:
        wl.headers, wl.lens = wl.derive(rigs["empty"].translated)
    keys, owners = prefixes(S, L)
    up = wl.prog != "nat44_ingress"
    target = int(owners[7])
    src_of_mac = {}
    for r in rigs.values():  # the same bindings everywhere: IPv4 frames are unaffected by an IPv6 address
        src_of_mac = bind_ipv6(r.dp, S, L)
    res_bound = len(src_of_mac)
    for s, r in rigs.items():
        share = {"p20": 0.2, "p50": 0.5}.get(s, 0.0)
        r.stage(to_ipv6(wl.headers, share, up, 11, src_of_mac) if share else wl.headers, wl.lens)
        r.li_cap = 1 << 19
        r.dp.acct_enable(wl.prog)
        r.dp.li_configure(0, r.li_cap)
        r.dp.li_target_set(target, 1)
        if s != "empty":
            assert r.dp.ipv6_prefixes_set(keys["addr"], keys["prefixlen"], owners) == 0
    res = {"frames": wl.n, "prog": wl.prog, "ipv6_bound_macs": res_bound, "mpps": {s: [] for s in SETTINGS},
           "li_records_per_batch": {}, "acct_packets_per_batch": {}}
    for s in SETTINGS:  # warm up every setting
        rigs[s].timed(2)
    for _ in range(rounds):
        for s in SETTINGS:
            mpps, recs = rigs[s].timed(steps)
            res["mpps"][s].append(round(mpps, 1))
            res["li_records_per_batch"][s] = int(np.median(recs)) if recs else 0
    for s in SETTINGS:
        r = rigs[s]
        r.dp.prof_enable(True)
        for _ in range(5):
            r.restore()
            r.step()
            r.dp.sync()
        prof = r.dp.prof_read()
        r.dp.prof_enable(False)
        r.restore()
        res["kernels_ms_" + s] = {k: round(v[1] / v[0], 4) for k, v in prof.items() if k.startswith(("k_acct", "k_li_capture"))}
        recs = r.dp.acct_dump()[1]
        res["acct_packets_per_batch"][s] = int(recs["up_packets"].sum() + recs["down_packets"].sum()) // max(r.step_no, 1)
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
