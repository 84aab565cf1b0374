// Tests of the host side of the DHCPv6 fast path (bng_dhcpv6_enable): ebpf::Loader's cache calls, shard::Route::ByValueMAC
// for dhcpv6_bindings (including a client re-bound under another MAC) and shard::Router::DHCPv6Enable
// (bng_host.hpp, bng_shard.hpp).  `test_dhcpv6_host cpu` needs no device: the routing table and NULL-context checks.
// `test_dhcpv6_host gpu` runs the calls against real contexts.
#include <array>
#include <cerrno>
#include <cstdio>
#include <string>

#include "../../bng_b200/host/bng_host.hpp"
#include "../../bng_b200/host/bng_shard.hpp"

using namespace bng;

static int g_fail = 0, g_checks = 0;
#define CHECK(c)                                                                \
    do {                                                                        \
        g_checks++;                                                             \
        if (!(c)) {                                                             \
            g_fail++;                                                           \
            fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #c);        \
        }                                                                       \
    } while (0)

static std::shared_ptr<Backend> open_ctx(uint32_t rank, uint32_t world) {
    bng_open_opts o{};
    o.struct_size = sizeof(o), o.device = -1, o.max_batch = 1 << 10, o.max_subscribers = 1 << 10;
    o.max_nat_sessions = 1 << 10, o.max_eim_mappings = 1 << 10, o.event_capacity = 1 << 10, o.world = world, o.rank = rank;
    auto b = Backend::Open(&o);
    if (!b->ctx) {
        fprintf(stderr, "FAIL bng_open: %s\n", b->open_error.c_str());
        g_fail++;
    }
    return b;
}

static bng_dhcpv6_binding binding(const std::array<uint8_t, 6> &mac, uint32_t iaid) {
    bng_dhcpv6_binding b{};
    memcpy(b.mac, mac.data(), 6);
    b.flags = BNG_DHCPV6_NA | BNG_DHCPV6_PD, b.pd_len = 56, b.iaid_na = iaid, b.iaid_pd = iaid + 1;
    b.preferred_lft = 3600, b.valid_lft = 7200, b.expires_s = 1u << 30;
    b.addr[0] = 0x20, b.addr[1] = 0x01, b.addr[15] = (uint8_t)iaid;
    b.prefix[0] = 0x20, b.prefix[1] = 0x01, b.prefix[5] = (uint8_t)iaid;
    return b;
}

static void cpu_checks() {
    CHECK(shard::RouteOf("dhcpv6_bindings") == shard::Route::ByValueMAC);
    CHECK(shard::RouteOf("dhcpv6_server_config") == shard::Route::Replicated);
    CHECK(shard::RouteOf("dhcpv6_stats") == shard::Route::Replicated);
    CHECK(bng_dhcpv6_enable(nullptr, 1) == -EINVAL);
    // routing by the value's MAC without a context: the owner is the MAC's shard
    auto dir = std::make_shared<shard::Directory>(8);
    shard::Router rt({}, dir);
    const std::array<uint8_t, 6> mac{0x02, 0x00, 0x00, 0x00, 0x00, 0x07};
    bng_dhcpv6_client_key k = ebpf::Loader::DHCPv6Key((const uint8_t *)"client-7", 8);
    bng_dhcpv6_binding b = binding(mac, 7);
    CHECK(rt.Owner("dhcpv6_bindings", &k, &b) == (int)dir->ShardOfMAC(shard::Directory::MacKey(mac.data())));
    CHECK(rt.Owner("dhcpv6_bindings", &k) == -ENOENT); // no shard holds it yet
}

static void gpu_checks() {
    // the Loader's calls on one context
    auto be = open_ctx(0, 1);
    if (!be->ctx) return;
    auto lr = ebpf::Loader::NewLoader("eth0", be);
    auto &l = **lr.value;
    CHECK(!l.Load());
    bng_dhcpv6_server_config cfg{};
    cfg.server_mac[0] = 0x02, cfg.duid_len = 10, cfg.dns_count = 1;
    CHECK(!l.SetDHCPv6ServerConfig(cfg));
    cfg.dns_count = 3;
    CHECK(l.SetDHCPv6ServerConfig(cfg)); // -EINVAL
    const std::array<uint8_t, 6> mac{0x02, 0x00, 0x00, 0x00, 0x00, 0x09};
    const uint8_t duid[10] = {0, 1, 0, 1, 1, 2, 3, 4, 5, 6};
    CHECK(!l.AddDHCPv6Binding(duid, 10, binding(mac, 9)));
    auto got = l.GetDHCPv6Binding(duid, 10); // staged: visible once applied (a lookup flushes)
    CHECK(!got.err && got.value->iaid_na == 9 && got.value->pd_len == 56);
    bng_dhcpv6_binding bad = binding(mac, 9);
    bad.flags = 0;
    CHECK(l.AddDHCPv6Binding(duid, 10, bad));
    CHECK(l.AddDHCPv6Binding(duid, 32, binding(mac, 9)));
    CHECK(!l.EnableDHCPv6FastPath(true));
    CHECK(!l.RemoveDHCPv6Binding(duid, 10));
    CHECK(l.GetDHCPv6Binding(duid, 10).err);

    // a Router of 4: bindings go to their MAC's shard, a re-bind under another MAC leaves the old one
    std::vector<std::shared_ptr<Backend>> shards;
    for (uint32_t r = 0; r < 4; r++) shards.push_back(open_ctx(r, 4));
    auto dir = std::make_shared<shard::Directory>(4);
    shard::Router rt(shards, dir);
    CHECK(rt.DHCPv6Enable(true) == 0);
    uint32_t zero = 0;
    cfg.dns_count = 2;
    CHECK(rt.Update("dhcpv6_server_config", &zero, &cfg) == 0);
    for (size_t s = 0; s < 4; s++) {
        bng_dhcpv6_server_config c2{};
        CHECK(bng_map_lookup(shards[s]->ctx, bng_map_id(shards[s]->ctx, "dhcpv6_server_config"), &zero, &c2) == 0 && c2.dns_count == 2);
    }
    bng_dhcpv6_client_key k = ebpf::Loader::DHCPv6Key(duid, 10);
    // two MACs on different shards
    std::array<uint8_t, 6> m1{0x02, 0, 0, 0, 0, 1}, m2 = m1;
    const uint32_t s1 = dir->ShardOfMAC(shard::Directory::MacKey(m1.data()));
    for (uint8_t i = 2; i < 250; i++) {
        m2[5] = i;
        if (dir->ShardOfMAC(shard::Directory::MacKey(m2.data())) != s1) break;
    }
    const uint32_t s2 = dir->ShardOfMAC(shard::Directory::MacKey(m2.data()));
    CHECK(s1 != s2);
    auto count = [&](size_t s) {
        bng_map_info mi{};
        bng_map_get_info(shards[s]->ctx, bng_map_id(shards[s]->ctx, "dhcpv6_bindings"), &mi);
        return mi.count;
    };
    const bng_dhcpv6_binding b1 = binding(m1, 1), b2 = binding(m2, 2);
    CHECK(rt.Update("dhcpv6_bindings", &k, &b1) == 0);
    CHECK(count(s1) == 1 && count(s2) == 0);
    CHECK(rt.Owner("dhcpv6_bindings", &k) == (int)s1);
    CHECK(rt.Update("dhcpv6_bindings", &k, &b2, BNG_ANY, true) == 0); // staged, re-bound
    CHECK(count(s1) == 0 && count(s2) == 1);
    bng_dhcpv6_binding v{};
    CHECK(rt.Lookup("dhcpv6_bindings", &k, &v) == 0 && v.iaid_na == 2);
    CHECK(rt.Delete("dhcpv6_bindings", &k) == 0);
    CHECK(count(s2) == 0);
    CHECK(rt.Lookup("dhcpv6_bindings", &k, &v) == -ENOENT);
    CHECK(rt.Delete("dhcpv6_bindings", &k) == -ENOENT);
}

int main(int argc, char **argv) {
    const std::string mode = argc > 1 ? argv[1] : "cpu";
    cpu_checks();
    if (mode == "gpu") gpu_checks();
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
