// Tests of the host side of Router and Neighbor Solicitations answered on the GPU (bng_nd_enable): slaac::BuildRA
// against byte vectors worked out by hand from pkg/slaac/radvd.go's buildRA, ebpf::Loader's ND calls,
// shard::Route::ByMAC for nd_bindings and shard::Router::NDEnable (bng_host.hpp, bng_shard.hpp).
// `test_nd_host cpu` needs no device: BuildRA, the routing table and the NULL-context check.  `test_nd_host gpu` runs
// the calls against real contexts.
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

static std::vector<uint8_t> unhex(const std::string &h) {
    std::vector<uint8_t> v;
    for (size_t i = 0; i + 1 < h.size(); i += 2) v.push_back((uint8_t)std::stoul(h.substr(i, 2), nullptr, 16));
    return v;
}
static std::vector<uint8_t> ip6(const char *hex) {
    return unhex(hex);
}
static slaac::Prefix prefix(const char *hex, uint8_t len) {
    slaac::Prefix p{};
    auto v = unhex(hex);
    memcpy(p.addr, v.data(), 16);
    p.len = len;
    return p;
}
static slaac::RouterConfig base() {
    slaac::RouterConfig rc;
    const uint8_t mac[6] = {0x02, 0xaa, 0xbb, 0xcc, 0xdd, 0x01};
    memcpy(rc.router_mac, mac, 6);
    auto ll = unhex("fe800000000000000000000000000001");
    memcpy(rc.router_ll, ll.data(), 16);
    return rc;
}
// head, tail of a built configuration, as hex
static bool ra_is(const bng_nd_config &c, const std::string &head, const std::string &tail) {
    const auto h = unhex(head), t = unhex(tail);
    if (c.ra_head_len != h.size() || c.ra_tail_len != t.size()) {
        fprintf(stderr, "lengths %u %u, want %zu %zu\n", c.ra_head_len, c.ra_tail_len, h.size(), t.size());
        return false;
    }
    if (memcmp(c.ra, h.data(), h.size()) || (t.size() && memcmp(c.ra + h.size(), t.data(), t.size()))) return false;
    for (size_t k = h.size() + t.size(); k < sizeof(c.ra); k++)
        if (c.ra[k]) return false;
    return true;
}

// buildRA's fields: type 134, code 0, checksum 0, curHopLimit 64, M|O flags, router lifetime (BE16), reachable time 0,
// retrans timer 0; SLLA {1, 1, mac}; MTU {5, 1, 0, 0, mtu}; each prefix {3, 4, len, L|A, 2592000, 604800, 0, prefix};
// RDNSS {25, 1 + 2n, 0, 0, 3 x lifetime, servers}; DNSSL {31, len, 0, 0, 3 x lifetime, labels, padding to 8}.
static void build_ra_checks() {
    const std::string slla = "0101" "02aabbccdd01";
    {   // no DNS, no shared prefix, Managed off, defaults (lifetime 1800 = 0x0708, no MTU)
        auto r = slaac::BuildRA(base());
        CHECK(r.ok());
        CHECK(ra_is(*r, "86000000" "40000708" "00000000" "00000000" + slla, ""));
        CHECK(r->router_mac[0] == 0x02 && r->router_ll[0] == 0xfe && r->router_ll[15] == 1);
    }
    {   // 2 DNS + 2 domains, 2 shared prefixes (the second given with host bits set), Managed and Other on, MTU 1500,
        // lifetime 600 (RDNSS / DNSSL lifetime 1800)
        auto rc = base();
        rc.managed = rc.other = true, rc.mtu = 1500, rc.default_lifetime = 600;
        rc.prefixes = {prefix("20010db8000100000000000000000000", 64), prefix("20010db80002ffff0000000000000001", 48)};
        rc.dns_servers = {ip6("20010db8000000000000000000000053"), ip6("20010db8000000000000000000000054"),
                          ip6("00000000000000000000ffffc0000201")}; // the IPv4-mapped one is dropped
        rc.dns_domains = {"isp.example", "example.net."};
        auto r = slaac::BuildRA(rc);
        CHECK(r.ok());
        const std::string head = "86000000" "40c00258" "00000000" "00000000" + slla + "05010000" "000005dc" +
                                 "03044080" "00278d00" "00093a80" "00000000" "20010db8000100000000000000000000" +
                                 "03043080" "00278d00" "00093a80" "00000000" "20010db8000200000000000000000000";
        const std::string tail = "19050000" "00000708" "20010db8000000000000000000000053" "20010db8000000000000000000000054" +
                                 std::string("1f050000" "00000708") + "03" "697370" "07" "6578616d706c65" "00" + "07" +
                                 "6578616d706c65" "03" "6e6574" "00" + "000000000000";
        CHECK(ra_is(*r, head, tail));
    }
    {   // 2 shared prefixes with Managed off: L and A
        auto rc = base();
        rc.prefixes = {prefix("20010db8000100000000000000000000", 64), prefix("20010db8000200000000000000000000", 56)};
        auto r = slaac::BuildRA(rc);
        CHECK(r.ok());
        CHECK(ra_is(*r, "86000000" "40000708" "00000000" "00000000" + slla +
                            "030440c0" "00278d00" "00093a80" "00000000" "20010db8000100000000000000000000" +
                            "030438c0" "00278d00" "00093a80" "00000000" "20010db8000200000000000000000000",
                    ""));
    }
    {   // a single DNS server, Managed on, no prefixes
        auto rc = base();
        rc.managed = true;
        rc.dns_servers = {ip6("20010db8000000000000000000000053")};
        auto r = slaac::BuildRA(rc);
        CHECK(r.ok());
        CHECK(ra_is(*r, "86000000" "40800708" "00000000" "00000000" + slla,
                    "19030000" "00001518" "20010db8000000000000000000000053"));
    }
    {   // more than nd_config holds: 9 shared prefixes (16 + 8 + 288 bytes)
        auto rc = base();
        for (int i = 0; i < 9; i++) rc.prefixes.push_back(prefix("20010db8000100000000000000000000", 64));
        CHECK(!slaac::BuildRA(rc).ok());
        rc.prefixes.pop_back(); // 8: 280 bytes
        CHECK(slaac::BuildRA(rc).ok());
    }
}

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

static bng_nd_binding binding(uint8_t i) {
    bng_nd_binding b{};
    b.prefix[0] = 0x20, b.prefix[1] = 0x01, b.prefix[7] = i;
    b.prefix_len = 64, b.pio_flags = BNG_ND_PIO_L | BNG_ND_PIO_A, b.valid_lft = 7200, b.preferred_lft = 3600;
    b.expires_s = 1u << 30;
    return b;
}

static void cpu_checks() {
    build_ra_checks();
    CHECK(shard::RouteOf("nd_bindings") == shard::Route::ByMAC);
    CHECK(shard::RouteOf("nd_config") == shard::Route::Replicated);
    CHECK(shard::RouteOf("nd_stats") == shard::Route::Replicated);
    CHECK(bng_nd_enable(nullptr, 1) == -EINVAL);
    auto dir = std::make_shared<shard::Directory>(8);
    shard::Router rt({}, dir);
    const uint8_t mac[6] = {0x02, 0, 0, 0, 0, 7};
    const uint64_t k = shard::Directory::MacKey(mac);
    CHECK(rt.Owner("nd_bindings", &k) == (int)dir->ShardOfMAC(k));
}

static void gpu_checks() {
    auto be = open_ctx(0, 1);
    if (!be->ctx) return;
    auto lr = ebpf::Loader::NewLoader("eth0", be);
    auto &l = **lr.value;
    CHECK(!l.Load());
    auto rc = base();
    rc.prefixes = {prefix("20010db8000100000000000000000000", 64)};
    rc.dns_servers = {ip6("20010db8000000000000000000000053")};
    rc.dns_domains = {"isp.example"};
    auto cfg = slaac::BuildRA(rc);
    CHECK(cfg.ok());
    CHECK(!l.SetNDConfig(*cfg)); // what BuildRA makes passes the update's checks
    bng_nd_config bad = *cfg;
    bad.ra[0] = 133;
    CHECK(l.SetNDConfig(bad));
    bad = *cfg;
    bad.router_ll[0] = 0x20;
    CHECK(l.SetNDConfig(bad));
    const uint8_t mac[6] = {0x02, 0, 0, 0, 0, 9};
    const uint64_t mk = shard::Directory::MacKey(mac);
    CHECK(!l.AddNDBinding(mk, binding(9)));
    auto got = l.GetNDBinding(mk); // staged: visible once applied (a lookup flushes)
    CHECK(!got.err && got.value->prefix[7] == 9 && got.value->prefix_len == 64);
    bng_nd_binding b = binding(9);
    b.pio_flags = 0x20;
    CHECK(l.AddNDBinding(mk, b));
    b = binding(9);
    b.prefix[15] = 1; // past /64
    CHECK(l.AddNDBinding(mk, b));
    CHECK(!l.EnableNDFastPath(true));
    CHECK(!l.EnableNDFastPath(false));
    CHECK(!l.RemoveNDBinding(mk));
    CHECK(l.GetNDBinding(mk).err);

    // a Router of 4: the configuration on every shard, a binding on its MAC's shard
    std::vector<std::shared_ptr<Backend>> shards;
    for (uint32_t r = 0; r < 4; r++) shards.push_back(open_ctx(r, 4));
    auto dir = std::make_shared<shard::Directory>(4);
    shard::Router rt(shards, dir);
    CHECK(rt.NDEnable(true) == 0);
    uint32_t zero = 0;
    CHECK(rt.Update("nd_config", &zero, &*cfg) == 0);
    for (size_t s = 0; s < 4; s++) {
        bng_nd_config c2{};
        CHECK(bng_map_lookup(shards[s]->ctx, bng_map_id(shards[s]->ctx, "nd_config"), &zero, &c2) == 0 &&
              !memcmp(&c2, &*cfg, sizeof(c2)));
    }
    auto count = [&](size_t s) {
        bng_map_info mi{};
        bng_map_get_info(shards[s]->ctx, bng_map_id(shards[s]->ctx, "nd_bindings"), &mi);
        return mi.count;
    };
    for (uint8_t i = 1; i <= 16; i++) {
        const uint8_t m[6] = {0x02, 0, 0, 0, 1, i};
        const uint64_t k = shard::Directory::MacKey(m);
        const bng_nd_binding v = binding(i);
        CHECK(rt.Update("nd_bindings", &k, &v, BNG_ANY, true) == 0);
    }
    uint32_t total = 0;
    for (size_t s = 0; s < 4; s++) total += count(s);
    CHECK(total == 16);
    for (uint8_t i = 1; i <= 16; i++) {
        const uint8_t m[6] = {0x02, 0, 0, 0, 1, i};
        const uint64_t k = shard::Directory::MacKey(m);
        bng_nd_binding v{};
        const size_t s = dir->ShardOfMAC(k);
        CHECK(bng_map_lookup(shards[s]->ctx, bng_map_id(shards[s]->ctx, "nd_bindings"), &k, &v) == 0 && v.prefix[7] == i);
        CHECK(rt.Delete("nd_bindings", &k) == 0);
    }
    total = 0;
    for (size_t s = 0; s < 4; s++) total += count(s);
    CHECK(total == 0);
}

int main(int argc, char **argv) {
    const std::string mode = argc > 1 ? argv[1] : "cpu";
    cpu_checks();
    if (mode == "gpu") gpu_checks();
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
