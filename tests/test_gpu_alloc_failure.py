"""A device allocation the driver refuses fails only the call that asked for it: bng_map_dump with a capacity whose
scratch cannot exist returns -ENOMEM, and the next batch on the same context runs as on a context that never saw the
failure (the refused allocation's error is not reported by that batch's launches)."""
import errno

import numpy as np
import pytest

from bng_b200 import layouts as L
from bng_b200 import synth as S

pytestmark = pytest.mark.gpu

N_SUBS = 64


def _dp():
    from bng_b200 import Dataplane
    return Dataplane(max_subscribers=1 << 10, max_nat_sessions=1 << 10, max_eim_mappings=1 << 10, max_batch=1 << 10)


def _provision(dp, keys, vals):
    cfg = np.zeros(1, L.antispoof_config)
    cfg["default_mode"] = 1  # strict: frames of unknown MACs are dropped
    assert dp.update("antispoof_config", np.uint32(0), cfg) == 0
    assert dp.update_batch("subscriber_bindings", keys, vals) == 0


def _batch():
    # bound subscribers with their own address, bound subscribers with another's, and unknown MACs
    sub = np.concatenate([np.arange(N_SUBS), np.arange(N_SUBS), np.arange(N_SUBS, 2 * N_SUBS)])
    src = S.sub_ip(sub)
    src[N_SUBS:2 * N_SUBS] = S.sub_ip((np.arange(N_SUBS) + 1) % N_SUBS)
    lens = np.full(sub.size, 64, np.uint32)
    hdr = S.ipv4_headers(S.sub_mac_key(sub), np.uint64(0x02FFFFFFFFFE), src, np.uint32(0x08080808), 6, 4000, 443, lens)
    return hdr.reshape(-1).copy(), lens


def test_refused_dump_scratch_leaves_the_next_batch_alone():
    keys, vals = S.bindings(N_SUBS)
    dp, ref = _dp(), _dp()
    try:
        for d in (dp, ref):
            _provision(d, keys, vals)
        # 2^40 entries of 8-byte keys: no device has the scratch, and the driver refuses it outright.  The host buffers
        # hold 4 entries; the call fails before it writes any.
        kbuf = np.full((4, 8), 0xA5, np.uint8)
        vbuf = np.full((4, 24), 0xA5, np.uint8)
        mid = dp.map_id("subscriber_bindings")
        r = dp.lib.bng_map_dump(dp.h, mid, kbuf.ctypes.data, vbuf.ctypes.data, 2**40)
        assert r == -errno.ENOMEM, r
        msg = dp.lib.bng_last_error(dp.h).decode()
        assert "dump" in msg and "memory" in msg, msg
        assert (kbuf == 0xA5).all() and (vbuf == 0xA5).all()

        pkts, lens = _batch()
        got = dp.run("antispoof_ingress", pkts.copy(), lens.copy(), 10**9, stride=64)
        want = ref.run("antispoof_ingress", pkts.copy(), lens.copy(), 10**9, stride=64)
        got, want = np.asarray(got), np.asarray(want)
        assert np.array_equal(got, want)
        assert (want[:N_SUBS] == 0).all() and (want[2 * N_SUBS:] != 0).all()  # passed and dropped frames alike

        k, v = dp.dump("subscriber_bindings")
        kr, vr = ref.dump("subscriber_bindings")
        assert len(k) == N_SUBS and np.array_equal(k, kr) and np.array_equal(v, vr)
    finally:
        dp.close()
        ref.close()
