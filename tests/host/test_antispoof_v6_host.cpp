// Tests of the host side of antispoof by delegated prefix (bng_antispoof_ipv6_prefixes_enable):
// antispoof::ManagerConfig::ValidateIPv6Prefixes applied by antispoof::Manager::Start, and
// shard::Router::AntispoofIPv6PrefixesEnable reaching every shard (bng_host.hpp, bng_shard.hpp).
// `test_antispoof_v6_host cpu` needs no device: the NULL-context check.  `test_antispoof_v6_host gpu` observes the
// flag through its effect: a strict binding's hosts in its delegated /56 are dropped with the flag off and allowed
// with it on.  Through the Router it also checks that a subscriber's binding (routed ByMAC) and its prefix (routed
// ByValueIP) land on one shard, the shard its frames are steered to.
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

static std::array<uint8_t, 6> mac_of(uint8_t s) { return {0x02, 0xA6, 0x00, 0x00, 0x01, s}; }
static uint32_t ip_key(uint8_t s) {
    const uint8_t ip[4] = {100, 64, 1, s};
    uint32_t k;
    memcpy(&k, ip, 4);
    return k;
}
// 2001:db8:<s>00::/56, delegated to subscriber s
static std::array<uint8_t, 16> prefix(uint8_t s) {
    std::array<uint8_t, 16> a{};
    a[0] = 0x20, a[1] = 0x01, a[2] = 0x0d, a[3] = 0xb8, a[4] = 0x00, a[5] = s;
    return a;
}
static antispoof::SubscriberBinding strict_binding(uint8_t s) {
    antispoof::SubscriberBinding b{};
    b.IPv4Addr = ip_key(s), b.IPv4Valid = 1, b.Mode = 1; // strict, no IPv6 address of its own
    return b;
}

// n IPv6 frames from subscriber s's MAC whose sources are hosts in its /56, through antispoof_ingress on c.
// Returns the frames dropped.
static int send_v6(bng_ctx *c, uint8_t s, uint32_t n = 50) {
    const auto m = mac_of(s);
    const auto p = prefix(s);
    std::vector<uint8_t> frames(n * 64);
    for (uint32_t i = 0; i < n; i++) {
        uint8_t *f = &frames[i * 64];
        memcpy(f + 6, m.data(), 6);
        f[12] = 0x86, f[13] = 0xDD, f[14] = 0x60, f[20] = 17, f[21] = 64;
        memcpy(f + 22, p.data(), 16);
        f[29] = (uint8_t)(i + 1), f[37] = (uint8_t)(i * 7 + 1);
    }
    std::vector<uint32_t> len(n, 64);
    std::vector<uint8_t> verdict(n);
    bng_batch bt{};
    bt.pkts = frames.data(), bt.len = len.data(), bt.verdict = verdict.data(), bt.n = n, bt.stride = 64;
    bt.mem = BNG_MEM_HOST, bt.arena_bytes = (uint32_t)(frames.size() / 16), bt.now_ns = 1000000000ull;
    CHECK(bng_prog_run(c, bng_prog_id(c, "antispoof_ingress"), &bt) == 0);
    int shot = 0;
    for (uint8_t v : verdict) shot += v == BNG_TC_ACT_SHOT;
    return shot;
}

static void test_null() {
    CHECK(bng_antispoof_ipv6_prefixes_enable(nullptr, 1) == -EINVAL && bng_antispoof_ipv6_prefixes_enable(nullptr, 0) == -EINVAL);
}

static void test_gpu_manager() {
    for (bool validate : {false, true}) {
        auto be = open_ctx(0, 1);
        if (!be->ctx) return;
        antispoof::ManagerConfig cfg;
        cfg.Interface = "eth0", cfg.Backend_ = be, cfg.DefaultMode = antispoof::ModeStrict, cfg.ValidateIPv6Prefixes = validate;
        auto m = antispoof::Manager::NewManager(cfg);
        CHECK(m.ok());
        const auto mac = mac_of(1);
        const uint64_t key = shard::Directory::MacKey(mac.data());
        const auto b = strict_binding(1);
        CHECK(bng_map_update(be->ctx, bng_map_id(be->ctx, "subscriber_bindings"), &key, &b, BNG_ANY) == 0);
        const auto p = prefix(1);
        CHECK(dualstack::SetPrefix(be->ctx, p.data(), 56, ip_key(1), false) == 0);
        CHECK(send_v6(be->ctx, 1) == 50); // NewManager alone applies nothing
        CHECK(!(*m)->Start());
        CHECK(send_v6(be->ctx, 1) == (validate ? 0 : 50));
    }
}

static void test_gpu_router(uint32_t world) {
    auto dir = std::make_shared<shard::Directory>(world);
    std::vector<std::shared_ptr<Backend>> shards;
    for (uint32_t k = 0; k < world; k++) {
        shards.push_back(open_ctx(k, world));
        if (!shards.back()->ctx) return;
    }
    shard::Router r(shards, dir);
    antispoof::Config cfg{};
    cfg.DefaultMode = 1, cfg.LogViolations = 1;
    const uint32_t zero = 0;
    CHECK(r.Update("antispoof_config", &zero, &cfg) == 0);
    const uint8_t n = 24;
    std::vector<uint32_t> used(world, 0);
    for (uint8_t s = 1; s <= n; s++) {
        const auto mac = mac_of(s);
        const uint64_t key = shard::Directory::MacKey(mac.data());
        dir->Learn(key, ip_key(s));
        const auto b = strict_binding(s);
        CHECK(r.Update("subscriber_bindings", &key, &b) == 0);
        bng_ipv6_prefix_key pk{};
        pk.prefixlen = 56;
        const auto p = prefix(s);
        memcpy(pk.addr, p.data(), 16);
        const uint32_t v = ip_key(s);
        CHECK(r.Update("subscriber_ipv6", &pk, &v) == 0);
        // the binding, the prefix and the frames all have one shard
        const int ob = r.Owner("subscriber_bindings", &key), op = r.Owner("subscriber_ipv6", &pk, &v);
        uint8_t frame[64] = {};
        memcpy(frame + 6, mac.data(), 6);
        CHECK(ob >= 0 && ob == op && (uint32_t)ob == dir->SteerUpstream(frame, sizeof frame));
        if (ob >= 0 && ob < (int)world) used[ob]++;
    }
    uint32_t shards_used = 0;
    for (uint32_t u : used) shards_used += u != 0;
    CHECK(shards_used >= 2); // (the subscribers are spread over several shards)
    auto run_all = [&](int want) {
        for (uint8_t s = 1; s <= n; s++) {
            const auto mac = mac_of(s);
            const uint32_t k = dir->ShardOfMAC(shard::Directory::MacKey(mac.data()));
            CHECK(send_v6(shards[k]->ctx, s) == want);
        }
    };
    run_all(50); // off by default
    CHECK(r.AntispoofIPv6PrefixesEnable(true) == 0);
    run_all(0);
    CHECK(r.AntispoofIPv6PrefixesEnable(false) == 0);
    run_all(50);
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    test_null();
    if (mode == "gpu") {
        test_gpu_manager();
        test_gpu_router(2);
        test_gpu_router(8);
    }
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
