"""Which kernel instantiations a program launches, and under which profile names, for every combination of the
opt-in switches it reads.  The names are what bng_prof_read returns and what bench.py reports in kernels_ms, so the
table below pins them byte for byte, together with the number of launches of one batch.  It was recorded on an H100.

subscriber_ipv6 holds a prefix throughout, except in one run per program that has a switch gated by a table: there the
switch is on, the table is empty, and the run must launch what the run with the switch off launches."""
import itertools

import numpy as np
import pytest

import test_gpu_dhcpv6 as D6
import test_gpu_nd as ND
from bng_b200 import Dataplane
from bng_b200 import synth as S

ACCT_IDLE = ("off", "acct", "idle", "both")
B = (0, 1)
# per program: its switches and their values, in the order of the table's keys
SWITCHES = {
    "antispoof_ingress": (("as6", B),),
    "qos_egress_prog": (("qos6", B), ("acct_idle", ACCT_IDLE), ("li", B)),
    "qos_ingress_prog": (("qos6", B), ("acct_idle", ACCT_IDLE), ("li", B)),
    "nat44_egress": (("icmp", B), ("acct_idle", ACCT_IDLE), ("li", B)),
    "nat44_ingress": (("icmp", B), ("acct_idle", ACCT_IDLE), ("li", B)),
    "dhcp_fastpath_prog": (("dhcpv6", B), ("nd", B)),
    "pipeline_up": (("qos6", B), ("as6", B), ("icmp", B), ("acct_idle", ACCT_IDLE), ("li", B)),
    "pipeline_tc": (("qos6", B), ("as6", B), ("icmp", B), ("acct_idle", ACCT_IDLE), ("li", B)),
}
# the switch turned on over an empty table (subscriber_ipv6; dhcpv6_bindings for dhcp_fastpath_prog)
EMPTY = {"antispoof_ingress": "as6", "qos_egress_prog": "qos6", "qos_ingress_prog": "qos6",
         "dhcp_fastpath_prog": "dhcpv6", "pipeline_up": "as6", "pipeline_tc": "qos6"}
N_SUBS = 8
LI_ADDR = int(np.frombuffer(S.ip_bytes(S.sub_ip(3)).tobytes(), "<u4")[0])


def _batch():
    """64 UDP frames of 64 bytes from N_SUBS subscribers, stride 64."""
    i = np.arange(64)
    h = S.ipv4_headers(S.sub_mac_key(i % N_SUBS), 0x02FFFFFFFFFE, S.sub_ip(i % N_SUBS), 0x08080808, 17, 1000 + i, 53,
                       np.full(64, 64))
    return h.reshape(-1).copy(), np.full(64, 64, np.uint32)


def _set(dp, prog, sw, v):
    if sw == "as6":
        dp.antispoof_ipv6_prefixes_enable(v)
    elif sw == "qos6":
        dp.qos_ipv6_enable(v)
    elif sw == "icmp":
        (dp.nat_icmp_errors_enable if prog == "nat44_ingress" else dp.nat_icmp_errors_egress_enable)(v)
    elif sw == "acct_idle":
        dp.acct_enable(prog, v in ("acct", "both"))
        dp.idle_enable(prog, v in ("idle", "both"))
    elif sw == "li":
        if v:
            dp.li_target_set(LI_ADDR, 7)
        else:
            dp.li_target_del(LI_ADDR)
    elif sw == "dhcpv6":
        dp.dhcpv6_enable(v)
    elif sw == "nd":
        dp.nd_enable(v)


def _observe(dp, prog, combo):
    """(launches, sorted profile names) of one batch of prog with the switches set to combo."""
    for (sw, _), v in zip(SWITCHES[prog], combo):
        _set(dp, prog, sw, v)
    arena, lens = _batch()
    dp.prof_enable(True)
    n0 = dp.launch_count
    dp.run(prog, arena, lens, 2_000_000 * 10**9, stride=64)
    return dp.launch_count - n0, tuple(sorted(dp.prof_read()))


def observed(prog):
    """({combo: (launches, names)} over the product of prog's switches, the empty-table run's (launches, names))."""
    dp = Dataplane(max_batch=1 << 12)
    try:
        dp.li_configure(0, 1 << 12)
        off = tuple(vals[0] for _, vals in SWITCHES[prog])
        if prog == "dhcp_fastpath_prog":
            D6.gpu_setup(dp, D6.config(), {}, on=False)
            ND.gpu_setup(dp, ND.config(), {}, on=False)
        empty = None
        if prog in EMPTY:
            empty = _observe(dp, prog, tuple(1 if sw == EMPTY[prog] else v for (sw, _), v in zip(SWITCHES[prog], off)))
        if prog == "dhcp_fastpath_prog":
            D6.gpu_setup(dp, None, {S.dhcpv6_duid(1): D6.Binding(bytes.fromhex("020000000001"))}, on=False)
        else:
            pfx = bytes.fromhex("20010db8000100000000000000000000")
            assert dp.ipv6_prefixes_set([pfx], [64], np.array([LI_ADDR], "<u4")) == 0
        got = {c: _observe(dp, prog, c) for c in itertools.product(*(vals for _, vals in SWITCHES[prog]))}
        return got, empty
    finally:
        dp.close()


@pytest.mark.gpu
@pytest.mark.parametrize("prog", list(SWITCHES))
def test_variants(prog):
    got, empty = observed(prog)
    want = TABLE[prog]
    assert sorted(got) == sorted(want)
    for c in want:
        assert got[c] == want[c], f"{prog} {c}: {got[c]} vs {want[c]}"
    if empty is not None:
        off = tuple(vals[0] for _, vals in SWITCHES[prog])
        assert empty == want[off], f"{prog}: {EMPTY[prog]} on over an empty table: {empty} vs {want[off]}"


TABLE = {
    "antispoof_ingress": {
        (0,): (1, ("k_antispoof",)),
        (1,): (1, ("k_antispoof<v6>",)),
    },
    "qos_egress_prog": {
        (0, "off", 0): (12, ("(k_resolve<false, true, true>)", "group_by_key", "k_qos_classify")),
        (0, "off", 1): (13, (
            "(k_resolve<false, true, true>)", "group_by_key", "k_li_capture<down,v6>", "k_qos_classify",
        )),
        (0, "acct", 0): (13, ("(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_qos_classify")),
        (0, "acct", 1): (14, (
            "(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_li_capture<down,v6>", "k_qos_classify",
        )),
        (0, "idle", 0): (13, ("(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_qos_classify")),
        (0, "idle", 1): (14, (
            "(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_li_capture<down,v6>", "k_qos_classify",
        )),
        (0, "both", 0): (13, ("(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_qos_classify")),
        (0, "both", 1): (14, (
            "(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_li_capture<down,v6>", "k_qos_classify",
        )),
        (1, "off", 0): (12, ("(k_resolve<false, true, true>)", "group_by_key", "k_qos_classify<v6>")),
        (1, "off", 1): (13, (
            "(k_resolve<false, true, true>)", "group_by_key", "k_li_capture<down,v6>", "k_qos_classify<v6>",
        )),
        (1, "acct", 0): (13, ("(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_qos_classify<v6>")),
        (1, "acct", 1): (14, (
            "(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_li_capture<down,v6>",
            "k_qos_classify<v6>",
        )),
        (1, "idle", 0): (13, ("(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_qos_classify<v6>")),
        (1, "idle", 1): (14, (
            "(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_li_capture<down,v6>",
            "k_qos_classify<v6>",
        )),
        (1, "both", 0): (13, ("(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_qos_classify<v6>")),
        (1, "both", 1): (14, (
            "(k_resolve<false, true, true>)", "group_by_key", "k_acct<v6>", "k_li_capture<down,v6>",
            "k_qos_classify<v6>",
        )),
    },
    "qos_ingress_prog": {
        (0, "off", 0): (12, ("(k_resolve<false, true, false>)", "group_by_key", "k_qos_classify")),
        (0, "off", 1): (14, (
            "(k_resolve<false, true, false>)", "group_by_key", "k_li_capture<up,v6>", "k_li_verdict", "k_qos_classify",
        )),
        (0, "acct", 0): (13, ("(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_qos_classify")),
        (0, "acct", 1): (15, (
            "(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
            "k_qos_classify",
        )),
        (0, "idle", 0): (13, ("(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_qos_classify")),
        (0, "idle", 1): (15, (
            "(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
            "k_qos_classify",
        )),
        (0, "both", 0): (13, ("(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_qos_classify")),
        (0, "both", 1): (15, (
            "(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
            "k_qos_classify",
        )),
        (1, "off", 0): (12, ("(k_resolve<false, true, false>)", "group_by_key", "k_qos_classify<v6>")),
        (1, "off", 1): (14, (
            "(k_resolve<false, true, false>)", "group_by_key", "k_li_capture<up,v6>", "k_li_verdict",
            "k_qos_classify<v6>",
        )),
        (1, "acct", 0): (13, ("(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_qos_classify<v6>")),
        (1, "acct", 1): (15, (
            "(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
            "k_qos_classify<v6>",
        )),
        (1, "idle", 0): (13, ("(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_qos_classify<v6>")),
        (1, "idle", 1): (15, (
            "(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
            "k_qos_classify<v6>",
        )),
        (1, "both", 0): (13, ("(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_qos_classify<v6>")),
        (1, "both", 1): (15, (
            "(k_resolve<false, true, false>)", "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
            "k_qos_classify<v6>",
        )),
    },
    "nat44_egress": {
        (0, "off", 0): (12, ("(k_pipe_classify<false, false>)", "(k_resolve<true, false, false>)", "group_by_key")),
        (0, "off", 1): (14, (
            "(k_pipe_classify<false, false>)", "(k_resolve<true, false, false>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, "acct", 0): (13, (
            "(k_pipe_classify<false, false, false, true>)", "(k_resolve<true, false, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, "acct", 1): (15, (
            "(k_pipe_classify<false, false, false, true>)", "(k_resolve<true, false, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, "idle", 0): (13, (
            "(k_pipe_classify<false, false, false, true>)", "(k_resolve<true, false, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, "idle", 1): (15, (
            "(k_pipe_classify<false, false, false, true>)", "(k_resolve<true, false, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, "both", 0): (13, (
            "(k_pipe_classify<false, false, false, true>)", "(k_resolve<true, false, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, "both", 1): (15, (
            "(k_pipe_classify<false, false, false, true>)", "(k_resolve<true, false, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, "off", 0): (12, (
            "(k_pipe_classify<false, false, icmperr>)", "(k_resolve<true, false, false, icmperr>)", "group_by_key",
        )),
        (1, "off", 1): (14, (
            "(k_pipe_classify<false, false, icmperr>)", "(k_resolve<true, false, false, icmperr>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, "acct", 0): (13, (
            "(k_pipe_classify<false, false, false, true, icmperr>)", "(k_resolve<true, false, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, "acct", 1): (15, (
            "(k_pipe_classify<false, false, false, true, icmperr>)", "(k_resolve<true, false, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, "idle", 0): (13, (
            "(k_pipe_classify<false, false, false, true, icmperr>)", "(k_resolve<true, false, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, "idle", 1): (15, (
            "(k_pipe_classify<false, false, false, true, icmperr>)", "(k_resolve<true, false, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, "both", 0): (13, (
            "(k_pipe_classify<false, false, false, true, icmperr>)", "(k_resolve<true, false, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, "both", 1): (15, (
            "(k_pipe_classify<false, false, false, true, icmperr>)", "(k_resolve<true, false, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
    },
    "nat44_ingress": {
        (0, "off", 0): (1, ("k_nat_ingress",)),
        (0, "off", 1): (2, ("k_li_capture<down,v6>", "k_nat_ingress")),
        (0, "acct", 0): (2, ("k_acct<v6>", "k_nat_ingress")),
        (0, "acct", 1): (3, ("k_acct<v6>", "k_li_capture<down,v6>", "k_nat_ingress")),
        (0, "idle", 0): (2, ("k_acct<v6>", "k_nat_ingress")),
        (0, "idle", 1): (3, ("k_acct<v6>", "k_li_capture<down,v6>", "k_nat_ingress")),
        (0, "both", 0): (2, ("k_acct<v6>", "k_nat_ingress")),
        (0, "both", 1): (3, ("k_acct<v6>", "k_li_capture<down,v6>", "k_nat_ingress")),
        (1, "off", 0): (1, ("k_nat_ingress<icmperr>",)),
        (1, "off", 1): (2, ("k_li_capture<down,v6>", "k_nat_ingress<icmperr>")),
        (1, "acct", 0): (2, ("k_acct<v6>", "k_nat_ingress<icmperr>")),
        (1, "acct", 1): (3, ("k_acct<v6>", "k_li_capture<down,v6>", "k_nat_ingress<icmperr>")),
        (1, "idle", 0): (2, ("k_acct<v6>", "k_nat_ingress<icmperr>")),
        (1, "idle", 1): (3, ("k_acct<v6>", "k_li_capture<down,v6>", "k_nat_ingress<icmperr>")),
        (1, "both", 0): (2, ("k_acct<v6>", "k_nat_ingress<icmperr>")),
        (1, "both", 1): (3, ("k_acct<v6>", "k_li_capture<down,v6>", "k_nat_ingress<icmperr>")),
    },
    "dhcp_fastpath_prog": {
        (0, 0): (1, ("k_dhcp_fastpath",)),
        (0, 1): (1, ("k_dhcp_fastpath<nd>",)),
        (1, 0): (1, ("k_dhcp_fastpath<v6>",)),
        (1, 1): (1, ("k_dhcp_fastpath<v6,nd>",)),
    },
    "pipeline_up": {
        (0, 0, 0, "off", 0): (12, ("(k_pipe_classify<true, true>)", "(k_resolve<true, true, false>)", "group_by_key")),
        (0, 0, 0, "off", 1): (14, (
            "(k_pipe_classify<true, true, false, true>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 0, "acct", 0): (13, (
            "(k_pipe_classify<true, true, false, true>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 0, 0, "acct", 1): (15, (
            "(k_pipe_classify<true, true, false, true>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 0, "idle", 0): (13, (
            "(k_pipe_classify<true, true, false, true>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 0, 0, "idle", 1): (15, (
            "(k_pipe_classify<true, true, false, true>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 0, "both", 0): (13, (
            "(k_pipe_classify<true, true, false, true>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 0, 0, "both", 1): (15, (
            "(k_pipe_classify<true, true, false, true>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 1, "off", 0): (12, (
            "(k_pipe_classify<true, true, icmperr>)", "(k_resolve<true, true, false, icmperr>)", "group_by_key",
        )),
        (0, 0, 1, "off", 1): (14, (
            "(k_pipe_classify<true, true, false, true, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 1, "acct", 0): (13, (
            "(k_pipe_classify<true, true, false, true, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 0, 1, "acct", 1): (15, (
            "(k_pipe_classify<true, true, false, true, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 1, "idle", 0): (13, (
            "(k_pipe_classify<true, true, false, true, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 0, 1, "idle", 1): (15, (
            "(k_pipe_classify<true, true, false, true, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 1, "both", 0): (13, (
            "(k_pipe_classify<true, true, false, true, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 0, 1, "both", 1): (15, (
            "(k_pipe_classify<true, true, false, true, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 0, "off", 0): (12, (
            "(k_pipe_classify<true, true, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
        )),
        (0, 1, 0, "off", 1): (14, (
            "(k_pipe_classify<true, true, false, true, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 0, "acct", 0): (13, (
            "(k_pipe_classify<true, true, false, true, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 1, 0, "acct", 1): (15, (
            "(k_pipe_classify<true, true, false, true, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 0, "idle", 0): (13, (
            "(k_pipe_classify<true, true, false, true, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 1, 0, "idle", 1): (15, (
            "(k_pipe_classify<true, true, false, true, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 0, "both", 0): (13, (
            "(k_pipe_classify<true, true, false, true, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 1, 0, "both", 1): (15, (
            "(k_pipe_classify<true, true, false, true, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 1, "off", 0): (12, (
            "(k_pipe_classify<true, true, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)", "group_by_key",
        )),
        (0, 1, 1, "off", 1): (14, (
            "(k_pipe_classify<true, true, false, true, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 1, "acct", 0): (13, (
            "(k_pipe_classify<true, true, false, true, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 1, 1, "acct", 1): (15, (
            "(k_pipe_classify<true, true, false, true, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 1, "idle", 0): (13, (
            "(k_pipe_classify<true, true, false, true, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 1, 1, "idle", 1): (15, (
            "(k_pipe_classify<true, true, false, true, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 1, "both", 0): (13, (
            "(k_pipe_classify<true, true, false, true, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 1, 1, "both", 1): (15, (
            "(k_pipe_classify<true, true, false, true, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 0, "off", 0): (12, (
            "(k_pipe_classify<true, true, v6>)", "(k_resolve<true, true, false>)", "group_by_key",
        )),
        (1, 0, 0, "off", 1): (14, (
            "(k_pipe_classify<true, true, false, true, v6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 0, "acct", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 0, 0, "acct", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 0, "idle", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 0, 0, "idle", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 0, "both", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 0, 0, "both", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 1, "off", 0): (12, (
            "(k_pipe_classify<true, true, v6, icmperr>)", "(k_resolve<true, true, false, icmperr>)", "group_by_key",
        )),
        (1, 0, 1, "off", 1): (14, (
            "(k_pipe_classify<true, true, false, true, v6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 1, "acct", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, 0, 1, "acct", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 1, "idle", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, 0, 1, "idle", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 1, "both", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, 0, 1, "both", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 0, "off", 0): (12, (
            "(k_pipe_classify<true, true, v6, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
        )),
        (1, 1, 0, "off", 1): (14, (
            "(k_pipe_classify<true, true, false, true, v6, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 0, "acct", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 1, 0, "acct", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 0, "idle", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 1, 0, "idle", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 0, "both", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 1, 0, "both", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6, as6>)", "(k_resolve<true, true, false>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 1, "off", 0): (12, (
            "(k_pipe_classify<true, true, v6, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key",
        )),
        (1, 1, 1, "off", 1): (14, (
            "(k_pipe_classify<true, true, false, true, v6, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 1, "acct", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, 1, 1, "acct", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 1, "idle", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, 1, 1, "idle", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 1, "both", 0): (13, (
            "(k_pipe_classify<true, true, false, true, v6, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, 1, 1, "both", 1): (15, (
            "(k_pipe_classify<true, true, false, true, v6, as6, icmperr>)", "(k_resolve<true, true, false, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
    },
    "pipeline_tc": {
        (0, 0, 0, "off", 0): (12, (
            "(k_pipe_classify<true, true, true>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
        )),
        (0, 0, 0, "off", 1): (14, (
            "(k_pipe_classify<true, true, true, true>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 0, "acct", 0): (13, (
            "(k_pipe_classify<true, true, true, true>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 0, 0, "acct", 1): (15, (
            "(k_pipe_classify<true, true, true, true>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 0, "idle", 0): (13, (
            "(k_pipe_classify<true, true, true, true>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 0, 0, "idle", 1): (15, (
            "(k_pipe_classify<true, true, true, true>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 0, "both", 0): (13, (
            "(k_pipe_classify<true, true, true, true>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 0, 0, "both", 1): (15, (
            "(k_pipe_classify<true, true, true, true>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 1, "off", 0): (12, (
            "(k_pipe_classify<true, true, true, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key",
        )),
        (0, 0, 1, "off", 1): (14, (
            "(k_pipe_classify<true, true, true, true, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 1, "acct", 0): (13, (
            "(k_pipe_classify<true, true, true, true, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 0, 1, "acct", 1): (15, (
            "(k_pipe_classify<true, true, true, true, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 1, "idle", 0): (13, (
            "(k_pipe_classify<true, true, true, true, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 0, 1, "idle", 1): (15, (
            "(k_pipe_classify<true, true, true, true, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 0, 1, "both", 0): (13, (
            "(k_pipe_classify<true, true, true, true, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 0, 1, "both", 1): (15, (
            "(k_pipe_classify<true, true, true, true, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 0, "off", 0): (12, (
            "(k_pipe_classify<true, true, true, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
        )),
        (0, 1, 0, "off", 1): (14, (
            "(k_pipe_classify<true, true, true, true, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 0, "acct", 0): (13, (
            "(k_pipe_classify<true, true, true, true, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 1, 0, "acct", 1): (15, (
            "(k_pipe_classify<true, true, true, true, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 0, "idle", 0): (13, (
            "(k_pipe_classify<true, true, true, true, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 1, 0, "idle", 1): (15, (
            "(k_pipe_classify<true, true, true, true, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 0, "both", 0): (13, (
            "(k_pipe_classify<true, true, true, true, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (0, 1, 0, "both", 1): (15, (
            "(k_pipe_classify<true, true, true, true, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 1, "off", 0): (12, (
            "(k_pipe_classify<true, true, true, as6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key",
        )),
        (0, 1, 1, "off", 1): (14, (
            "(k_pipe_classify<true, true, true, true, as6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 1, "acct", 0): (13, (
            "(k_pipe_classify<true, true, true, true, as6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 1, 1, "acct", 1): (15, (
            "(k_pipe_classify<true, true, true, true, as6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 1, "idle", 0): (13, (
            "(k_pipe_classify<true, true, true, true, as6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 1, 1, "idle", 1): (15, (
            "(k_pipe_classify<true, true, true, true, as6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (0, 1, 1, "both", 0): (13, (
            "(k_pipe_classify<true, true, true, true, as6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (0, 1, 1, "both", 1): (15, (
            "(k_pipe_classify<true, true, true, true, as6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 0, "off", 0): (12, (
            "(k_pipe_classify<true, true, true, v6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
        )),
        (1, 0, 0, "off", 1): (14, (
            "(k_pipe_classify<true, true, true, true, v6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 0, "acct", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 0, 0, "acct", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 0, "idle", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 0, 0, "idle", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 0, "both", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 0, 0, "both", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 1, "off", 0): (12, (
            "(k_pipe_classify<true, true, true, v6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key",
        )),
        (1, 0, 1, "off", 1): (14, (
            "(k_pipe_classify<true, true, true, true, v6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 1, "acct", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, 0, 1, "acct", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 1, "idle", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, 0, 1, "idle", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 0, 1, "both", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>",
        )),
        (1, 0, 1, "both", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 0, "off", 0): (12, (
            "(k_pipe_classify<true, true, true, v6, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
        )),
        (1, 1, 0, "off", 1): (14, (
            "(k_pipe_classify<true, true, true, true, v6, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 0, "acct", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 1, 0, "acct", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 0, "idle", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 1, 0, "idle", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 0, "both", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>",
        )),
        (1, 1, 0, "both", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6, as6>)", "(k_resolve<true, true, false, tc>)", "group_by_key",
            "k_acct<v6>", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 1, "off", 0): (12, (
            "(k_pipe_classify<true, true, true, v6, as6, icmperr>)", "(k_resolve<true, true, false, tc, icmperr>)",
            "group_by_key",
        )),
        (1, 1, 1, "off", 1): (14, (
            "(k_pipe_classify<true, true, true, true, v6, as6, icmperr>)",
            "(k_resolve<true, true, false, tc, icmperr>)", "group_by_key", "k_li_capture<up,v6>", "k_li_verdict",
        )),
        (1, 1, 1, "acct", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6, as6, icmperr>)",
            "(k_resolve<true, true, false, tc, icmperr>)", "group_by_key", "k_acct<v6>",
        )),
        (1, 1, 1, "acct", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6, as6, icmperr>)",
            "(k_resolve<true, true, false, tc, icmperr>)", "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>",
            "k_li_verdict",
        )),
        (1, 1, 1, "idle", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6, as6, icmperr>)",
            "(k_resolve<true, true, false, tc, icmperr>)", "group_by_key", "k_acct<v6>",
        )),
        (1, 1, 1, "idle", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6, as6, icmperr>)",
            "(k_resolve<true, true, false, tc, icmperr>)", "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>",
            "k_li_verdict",
        )),
        (1, 1, 1, "both", 0): (13, (
            "(k_pipe_classify<true, true, true, true, v6, as6, icmperr>)",
            "(k_resolve<true, true, false, tc, icmperr>)", "group_by_key", "k_acct<v6>",
        )),
        (1, 1, 1, "both", 1): (15, (
            "(k_pipe_classify<true, true, true, true, v6, as6, icmperr>)",
            "(k_resolve<true, true, false, tc, icmperr>)", "group_by_key", "k_acct<v6>", "k_li_capture<up,v6>",
            "k_li_verdict",
        )),
    },
}
