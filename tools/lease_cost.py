"""What the DHCP lease census and expiry sweep cost at the reference's capacities (1e6 subscriber_pools, 1e5
vlan_subscriber_pools, 1e6 circuit_id_subscribers and 1e6 circuit_id_map entries over 64 pools): the wall time of
bng_dhcp_lease_census and of bng_dhcp_lease_sweep with 0, 1 % and 100 % of the entries due, their kernels' times, and
the host alternative (bng_map_dump of the three lease maps plus one bng_map_delete per due entry, the deletes timed on a
sample).  The variants alternate in one process; the tables are reloaded before every sweep that removes.

    python tools/lease_cost.py [--subs 1000000] [--reps 5] [--sample 256] [--out FILE]

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

import subprocess  # noqa: E402

NS = 10**9
T0 = 1_000_000  # seconds: every lease expires after it; the due share is drawn below it


def sm_clock_now():
    """The SM clock as nvidia-smi reads it at this moment (a query only), or None."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        return q.strip()
    except Exception:
        return None


def tables(n, due_permille, seed=7):
    """[(map, keys, values)]: n subscribers by MAC and by circuit-id, n // 10 by VLAN pair, circuit_id_map for all."""
    from bng_b200 import layouts as L
    from bng_b200 import synth as S
    sub = np.arange(n, dtype=np.uint32)
    pa = np.zeros(n, L.pool_assignment)
    pa["pool_id"] = 1 + sub % 64
    pa["allocated_ip"] = S.ip_bytes(np.uint32(0x0A000000) + sub)
    due = (S.splitmix64_array(seed, n) % np.uint64(1000)).astype(np.int64) < due_permille
    pa["lease_expiry"] = np.where(due, T0 - 10, T0 + 3600)
    pools = np.zeros(64, L.ip_pool)
    pools["network"] = S.ip_bytes(np.uint32(0x0A000000) + (np.arange(64, dtype=np.uint32) << 14))
    pools["prefix_len"] = 8
    nv = max(n // 10, 1)
    vk = np.zeros(nv, L.vlan_key)
    vk["s_tag"], vk["c_tag"] = 1 + np.arange(nv) % 4000, 1 + np.arange(nv) // 4000
    ck = np.zeros((n, 32), np.uint8)
    ck[:, :8] = np.frombuffer(b"port-id:", np.uint8)
    ck[:, 8:12] = sub.view(np.uint8).reshape(-1, 4)
    mac = S.sub_mac_key(sub)
    return [("ip_pools", np.arange(1, 65, dtype="<u4"), pools), ("subscriber_pools", mac, pa),
            ("vlan_subscriber_pools", vk, pa[:nv]), ("circuit_id_subscribers", ck, pa),
            ("circuit_id_map", S.splitmix64_array(seed + 1, n), mac)]


def load(dp, ups):
    from bng_b200.layouts import as_bytes
    for m, k, v in ups:
        assert dp.update_batch(m, as_bytes(k), as_bytes(v)) == 0, m
    dp.sync()


def kernels(dp, fn, prefix="k_lease"):
    dp.prof_enable(True)
    fn()
    prof = dp.prof_read()
    dp.prof_enable(False)
    return {k: round(v[1] / v[0], 4) for k, v in prof.items() if k.startswith(prefix) or k.startswith("k_table_rebuild")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subs", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=256)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from bng_b200 import Dataplane
    from bng_b200.layouts import bng_lease_removed
    res = {"card": card(), "subscribers": a.subs}
    now = T0 * NS
    cap = 3 * a.subs
    out = np.zeros(cap, bng_lease_removed)
    for permille in (0, 10, 1000):
        dp = Dataplane(max_batch=1 << 10, max_nat_sessions=1 << 10, max_eim_mappings=1 << 10)  # the default 1e6 subscribers
        ups = tables(a.subs, permille)
        dp.lease_addr_order(True)  # synth.ip_bytes writes wire order
        load(dp, ups)
        r = {}
        dp.lease_census(now)  # scratch allocated
        ts = []
        for _ in range(a.reps):
            t = time.perf_counter()
            s = dp.lease_census(now)[0]
            ts.append((time.perf_counter() - t) * 1e3)
        for _ in range(200):  # the clock under this load: read right after a burst of censuses
            dp.lib.bng_dhcp_lease_sweep(dp.h, now, 0, None, 0, None)
        r["sm_clock_under_load"] = sm_clock_now()
        r["census"] = {"summary": s, "ms": [round(x, 3) for x in ts], "kernels_ms": kernels(dp, lambda: dp.lease_census(now))}
        ts = []
        for _ in range(a.reps):  # the dry run: the same pass, nothing removed
            t = time.perf_counter()
            found = dp.lib.bng_dhcp_lease_sweep(dp.h, now, 0, None, 0, None)
            ts.append((time.perf_counter() - t) * 1e3)
        r["dry_run"] = {"found": int(found), "ms": [round(x, 3) for x in ts]}
        # the host alternative: dump the three maps to find the due entries, then one delete per entry (a sample)
        t = time.perf_counter()
        dumps = {m: dp.dump(m) for m in ("subscriber_pools", "vlan_subscriber_pools", "circuit_id_subscribers")}
        dump_ms = (time.perf_counter() - t) * 1e3
        keys = dumps["subscriber_pools"][0][: a.sample]
        t = time.perf_counter()
        for k in keys:
            dp.delete("subscriber_pools", k)
        del_ms = (time.perf_counter() - t) * 1e3 / max(len(keys), 1)
        r["host"] = {"dump_ms": round(dump_ms, 1), "delete_ms_each": round(del_ms, 4),
                     "deletes_projected_ms": round(del_ms * found, 1)}
        load(dp, ups[1:2])  # the sampled entries back
        ts, rebuilds = [], dp.lease_table_rebuilds()
        for rep in range(a.reps):
            t = time.perf_counter()
            n = dp.lib.bng_dhcp_lease_sweep(dp.h, now, 0, out.ctypes.data, cap, None)
            ts.append((time.perf_counter() - t) * 1e3)
            assert n == found, (n, found)
            if permille:
                load(dp, ups[1:])
        r["sweep"] = {"removed": int(found), "ms": [round(x, 3) for x in ts],
                      "rebuilds_per_sweep": (dp.lease_table_rebuilds() - rebuilds) / a.reps}
        r["sweep_kernels_ms"] = kernels(dp, lambda: dp.lib.bng_dhcp_lease_sweep(dp.h, now, 0, out.ctypes.data, cap, None))
        res[f"due_{permille}_permille"] = r
        dp.close()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
