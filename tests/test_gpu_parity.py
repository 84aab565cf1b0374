"""GPU parity: the CUDA dataplane, driven through the C ABI, against the CPU
oracle(s) and the committed golden vectors, bit for bit.  Every script runs
three times: with pageable host buffers (whole-arena staging copies), with pinned
host buffers (zero-copy header gather/scatter pipeline) and with device-resident
buffers (BNG_MEM_DEVICE, synchronised through torch only, as its callers do)."""
import os

import pytest

import harness
import scenarios

pytestmark = pytest.mark.gpu
FEEDS = [False, True, "device"]
FEED_IDS = ["pageable", "pinned", "device"]
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def gpu_results():
    cache = {}

    def get(script, pinned):
        if (script, pinned) not in cache:
            be = harness.GpuBackend(pinned=pinned)
            try:
                cache[(script, pinned)] = harness.run_script(be, scenarios.ALL_SCRIPTS[script]())
            finally:
                be.close()
        return cache[(script, pinned)]

    return get


@pytest.mark.parametrize("pinned", FEEDS, ids=FEED_IDS)
@pytest.mark.parametrize("script", sorted(scenarios.ALL_SCRIPTS))
def test_gpu_matches_golden(script, pinned, gpu_results):
    gold = harness.load_golden(os.path.join(GOLD, script + ".npz"))
    harness.compare(gold, gpu_results(script, pinned), f"{script}: golden vs gpu ({FEED_IDS[FEEDS.index(pinned)]})")


@pytest.mark.parametrize("script", ["pipeline", "nat", "dhcp"])
def test_gpu_matches_golden_abi_host_arena(script, gpu_results):
    """Frames in memory obtained from bng_host_alloc() (huge-page backed, cudaHostRegister'ed)."""
    gold = harness.load_golden(os.path.join(GOLD, script + ".npz"))
    harness.compare(gold, gpu_results(script, "abi"), f"{script}: golden vs gpu (bng_host_alloc arena)")


def _matches_live_oracle(script, pinned, ora_kind, gpu_results):
    if ora_kind == "none":
        pytest.fail("no oracle library present on this box")
    be = harness.OracleBackend(ora_kind)
    res = harness.run_script(be, scenarios.ALL_SCRIPTS[script]())
    harness.compare(res, gpu_results(script, pinned), f"{script}: {ora_kind} oracle vs gpu ({FEED_IDS[FEEDS.index(pinned)]})")


@pytest.mark.parametrize("script", sorted(scenarios.ALL_SCRIPTS))
def test_gpu_matches_live_oracle(script, ora_kind, gpu_results):
    _matches_live_oracle(script, False, ora_kind, gpu_results)


@pytest.mark.parametrize("pinned", FEEDS[1:], ids=FEED_IDS[1:])
@pytest.mark.parametrize("script", sorted(scenarios.ALL_SCRIPTS))
def test_gpu_matches_live_oracle_pinned_and_device(script, pinned, ora_kind, gpu_results):
    _matches_live_oracle(script, pinned, ora_kind, gpu_results)
