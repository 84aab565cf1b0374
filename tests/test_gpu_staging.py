"""The control-plane calls that move host arrays to the device and back in chunks, at their chunk edges: map updates,
lookups and dumps (2^18 items a chunk), accounting and idle reads (2^16), idle timeouts (2^18), the records a restore
loads (2^16), and hand-over exports whose staged regions are not multiples of 256 bytes."""
import errno

import numpy as np
import pytest

import harness
from bng_b200 import layouts as L
from bng_b200 import synth as S
from bng_b200 import workloads as W
from test_gpu_move import _load, _sections_equal, _words

pytestmark = pytest.mark.gpu

MAP_CHUNK, READ_CHUNK = 1 << 18, 1 << 16


def _dp(n):
    from bng_b200 import Dataplane
    return Dataplane(max_subscribers=max(n, 1024), max_batch=1 << 10)


def _keys(n):
    return S.ip_bytes(S.sub_ip(np.arange(n)))


def _rows(k, v):
    return sorted(bytes(r) for r in np.concatenate([k, harness.mask_padding("qos_ingress", v)], axis=1))


@pytest.mark.parametrize("n", [MAP_CHUNK - 1, MAP_CHUNK, MAP_CHUNK + 1, 2 * MAP_CHUNK + 1])
def test_map_update_lookup_dump(n):
    rng = np.random.Generator(np.random.PCG64(n))
    keys = _keys(n + 1)  # the last one is never inserted
    vals = rng.integers(0, 256, (n, L.token_bucket.itemsize), dtype=np.uint8)
    with _dp(2 * n) as dp:
        assert dp.update_batch("qos_ingress", keys[:n], vals) == 0
        assert _rows(*dp.dump("qos_ingress")) == _rows(keys[:n], vals)
        for i in sorted({0, MAP_CHUNK - 1, MAP_CHUNK, n // 2, n - 1} & set(range(n))):
            assert np.array_equal(harness.mask_padding("qos_ingress", dp.lookup("qos_ingress", keys[i]).reshape(1, -1)),
                                  harness.mask_padding("qos_ingress", vals[i:i + 1])), i
        # a miss leaves the caller's value as it was
        out = np.full(L.token_bucket.itemsize, 0xA5, np.uint8)
        r = dp.lib.bng_map_lookup(dp.h, dp.map_id("qos_ingress"), np.ascontiguousarray(keys[n]).ctypes.data, out.ctypes.data)
        assert r == -errno.ENOENT and (out == 0xA5).all()
        # BPF_NOEXIST over the old keys and as many new ones: the first error is reported, the new keys go in and the
        # old values stay
        more = _keys(2 * n)[n:]
        both = np.concatenate([keys[:n], more])
        vals2 = rng.integers(0, 256, (2 * n, L.token_bucket.itemsize), dtype=np.uint8)
        assert dp.update_batch("qos_ingress", both, vals2, flags=1) == -errno.EEXIST
        assert _rows(*dp.dump("qos_ingress")) == _rows(both, np.concatenate([vals, vals2[n:]]))


@pytest.mark.parametrize("n", [READ_CHUNK - 1, READ_CHUNK + 1, 2 * READ_CHUNK + 1, MAP_CHUNK + 1])
def test_acct_and_idle_reads(n):
    rng = np.random.Generator(np.random.PCG64(n))
    present = 3 * n // 4
    keys = _keys(n)
    perm = rng.permutation(n)  # the absent addresses are spread over every chunk
    with _dp(n) as dp:
        assert dp.update_batch("qos_ingress", keys[perm[:present]], np.zeros(present, L.token_bucket)) == 0
        dp.acct_enable("qos_ingress_prog")
        tos = rng.integers(1, 1 << 30, n).astype(np.uint32)
        found = dp.idle_timeout_set(keys, tos)
        inside = np.zeros(n, bool)
        inside[perm[:present]] = True
        assert np.array_equal(found, inside)
        a, recs = dp.acct_dump()
        assert len(a) == present
        r, f = dp.acct_read(keys)
        assert np.array_equal(f, inside)
        want = dict(zip(a.tolist(), [bytes(x) for x in recs.view(np.uint8).reshape(-1, 64)]))
        words = _words(keys)
        got = {int(w): bytes(x) for w, x, ok in zip(words, r.view(np.uint8).reshape(-1, 64), f) if ok}
        assert got == want
        assert (r[~f].view(np.uint8) == 0).all()
        ir, f2 = dp.idle_read(keys)
        assert np.array_equal(f2, inside)
        assert np.array_equal(ir["timeout_s"][inside], tos[inside]) and (ir[~inside].view(np.uint8) == 0).all()
        # the scan: the first one starts every record, the next finds all of them past a 1 s timeout, for a cap below
        # and above their count
        dp.idle_timeout_set(keys, 1)
        assert dp.idle_scan(10**15)[2] == 0
        for cap in (present - 1, present + 5):
            sa, srec, cnt = dp.idle_scan(10**15 + 10**10, cap=cap)
            assert cnt == present and len(sa) == min(present, cap)
            assert set(sa.tolist()) <= set(words[inside].tolist()) and (srec["timeout_s"] == 1).all()


@pytest.mark.parametrize("at", [MAP_CHUNK - 1, MAP_CHUNK])
def test_idle_timeout_repeated_across_a_chunk_edge(at):
    """An address given twice, on both sides of a chunk edge (or both in the last item of one chunk and the first of
    the next): the later value wins."""
    n = MAP_CHUNK + 8
    keys = _keys(n)
    with _dp(n) as dp:
        assert dp.update_batch("qos_ingress", keys, np.zeros(n, L.token_bucket)) == 0
        addrs = keys.copy()
        addrs[at + 1] = keys[at]
        addrs[n - 1] = keys[3]
        tos = np.arange(1, n + 1, dtype=np.uint32)
        assert dp.idle_timeout_set(addrs, tos).all()
        r, f = dp.idle_read(keys[[at, 3]])
        assert f.all() and r["timeout_s"].tolist() == [at + 2, n]


def test_snapshot_restore_of_many_records():
    n = 2 * READ_CHUNK + 1
    rng = np.random.Generator(np.random.PCG64(11))
    keys = _keys(n)
    with _dp(n) as dp, _dp(n) as twin:
        assert dp.update_batch("qos_ingress", keys, np.zeros(n, L.token_bucket)) == 0
        dp.acct_enable("qos_ingress_prog")
        tos = rng.integers(1, 1 << 30, n).astype(np.uint32)
        assert dp.idle_timeout_set(keys, tos).all()
        blob = bytearray(dp.snapshot())
        sec = {s.name: s for s in harness.blob_sections(blob)}
        acct = sec["subscriber_acct"]
        assert len(acct.keys) == n and len(sec["subscriber_idle"].keys) == n
        acct.vals[:] = rng.integers(0, 256, acct.vals.shape, dtype=np.uint8)  # written into the blob
        twin.restore(bytes(blob))
        a, recs = twin.acct_dump()
        want = sorted(zip(_words(acct.keys).tolist(), [bytes(v) for v in acct.vals]))
        assert sorted(zip(a.tolist(), [bytes(x) for x in recs.view(np.uint8).reshape(-1, 64)])) == want
        r, f = twin.idle_read(keys)
        assert f.all() and np.array_equal(r["timeout_s"], tos)


@pytest.mark.parametrize("acct_idle", [False, True], ids=["plain", "records"])
@pytest.mark.parametrize("v6_nd", [False, True], ids=["v4", "v6_nd"])
def test_sub_export_with_odd_region_sizes(acct_idle, v6_nd):
    """3 addresses and 5 MACs: every staged region ends off a 256-byte boundary."""
    from bng_b200 import Dataplane
    opts = dict(max_batch=1 << 14, max_subscribers=1 << 11, max_nat_sessions=1 << 14, max_eim_mappings=1 << 14)
    wl = W.pipeline(1 << 13, 0, 1, n_subs=40, flows_per_sub=8, imix=True)
    with Dataplane(**opts) as dp, Dataplane(**opts) as dst:
        _load(dp, wl)
        ips = _words(S.ip_bytes(S.sub_ip(np.arange(40))))
        if acct_idle:
            dp.acct_enable("pipeline_up")
            dp.idle_enable("pipeline_up")
            dp.idle_timeout_set(ips, 300)
        if v6_nd:
            v6 = np.zeros((20, 16), np.uint8)
            v6[:, :4] = [0x20, 0x01, 0x0D, 0xB8]
            v6[:, 5] = np.arange(20)
            assert dp.ipv6_prefixes_set(v6, [56] * 20, ips[:20]) == 0
            nd = np.zeros(20, L.bng_nd_binding)
            nd["prefix"], nd["prefix_len"], nd["pio_flags"] = v6, 64, 0xC0
            nd["valid_lft"], nd["preferred_lft"], nd["expires_s"] = 7200, 3600, 2_000_000
            assert dp.update_batch("nd_bindings", S.sub_mac_key(np.arange(20)), nd) == 0
        for p, h, l in wl.prewarm:
            dp.run(p, h.reshape(-1).copy(), l.copy(), wl.now0 - 1, stride=64)
        dp.run("pipeline_up", wl.headers.reshape(-1).copy(), wl.lens.copy(), wl.now0, stride=64)
        addrs = ips[[2, 9, 17]]
        macs = S.sub_mac_key(np.array([2, 9, 17, 30, 3000]))  # the last one has no entry
        blob = dp.sub_export(addrs, macs)
        assert dp.sub_import(dp.sub_export(addrs, macs, detach=True)) == 0  # detach and take back
        _sections_equal(dp.sub_export(addrs, macs), blob)
        assert dst.sub_import(blob) == 0
        _sections_equal(dst.sub_export(addrs, macs), blob)
