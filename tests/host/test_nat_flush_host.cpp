// Tests of the host side of the NAT flow-state flush: the grouping of Router::NatFlush by owner shard and the
// broadcast of addresses without a known owner (bng_shard.hpp), and nat::Manager::FlushSessions (bng_host.hpp).
// `test_nat_flush_host cpu` needs no device; `test_nat_flush_host gpu` also creates one flow per subscriber on two
// dataplane contexts and flushes them through the router and the manager.
#include <cstdio>
#include <string>

#include "../../bng_b200/host/bng_host.hpp"
#include "../../bng_b200/host/bng_shard.hpp"

using namespace bng;

static int g_fail = 0, g_checks = 0;
#define CHECK_EQ(a, b)                                                                                        \
    do {                                                                                                      \
        g_checks++;                                                                                           \
        auto va = (a);                                                                                        \
        auto vb = (b);                                                                                        \
        if (!(va == vb)) {                                                                                    \
            g_fail++;                                                                                         \
            fprintf(stderr, "FAIL %s:%d: %s == %s (%llu vs %llu)\n", __FILE__, __LINE__, #a, #b,              \
                    (unsigned long long)va, (unsigned long long)vb);                                          \
        }                                                                                                     \
    } while (0)

static uint32_t key(uint8_t a, uint8_t b, uint8_t c, uint8_t d) { // the 4 key bytes as the maps hold them
    const uint8_t k[4] = {a, b, c, d};
    uint32_t v;
    memcpy(&v, k, 4);
    return v;
}

static uint64_t mac_of(uint32_t s) { return 0x020000000000ull + s * 0x10001ull; }

static void test_grouping() {
    for (uint32_t world : {2u, 8u}) {
        auto dir = std::make_shared<shard::Directory>(world);
        std::vector<std::shared_ptr<Backend>> shards;
        for (uint32_t i = 0; i < world; i++) shards.push_back(std::make_shared<Backend>()); // never opened
        shard::Router r(shards, dir);
        std::vector<uint32_t> addrs;
        for (uint32_t s = 0; s < 64; s++) {
            const uint32_t ip = key(10, 1, (uint8_t)(s >> 8), (uint8_t)s);
            dir->Learn(mac_of(s), ip);
            addrs.push_back(ip);
        }
        const uint32_t unknown = key(192, 0, 2, 1);
        addrs.push_back(unknown);
        addrs.push_back(addrs[5]); // a duplicate goes where its address goes
        auto g = r.NatFlushGroups(addrs.data(), addrs.size());
        CHECK_EQ(g.size(), (size_t)world);
        size_t total = 0;
        for (uint32_t k = 0; k < world; k++) {
            total += g[k].size();
            size_t unknown_seen = 0;
            for (uint32_t a : g[k]) {
                if (a == unknown) {
                    unknown_seen++;
                    continue;
                }
                auto s = dir->ShardOfIP(a);
                CHECK_EQ(s.has_value(), true);
                if (s) CHECK_EQ(*s, k); // every known address on its owner only
            }
            CHECK_EQ(unknown_seen, (size_t)1); // the address without an owner on every shard
        }
        CHECK_EQ(total, (size_t)64 + 1 + world);
        // every known address appears exactly as often as it was given
        for (uint32_t s = 0; s < 64; s++) {
            size_t seen = 0;
            for (auto &v : g)
                for (uint32_t a : v) seen += a == addrs[s];
            CHECK_EQ(seen, (size_t)(s == 5 ? 2 : 1));
        }
        // a forgotten subscriber has no owner any more: broadcast
        dir->Forget(mac_of(0));
        g = r.NatFlushGroups(addrs.data(), 1);
        for (auto &v : g) CHECK_EQ(v.size(), (size_t)1);
        // nothing to flush: no shard is called (the shards here are not open, a call would fail)
        CHECK_EQ(r.NatFlush(nullptr, 0, 1), 0);
        CHECK_EQ(r.NatFlush(nullptr, 3, 1), -EINVAL);
    }
}

// One 64-byte UDP frame from `src` (key bytes) to 8.8.8.8.
static void udp_frame(uint8_t *f, uint32_t src, uint16_t sport) {
    memset(f, 0, 64);
    f[12] = 0x08, f[14] = 0x45, f[16] = 0, f[17] = 50, f[22] = 64, f[23] = 17;
    memcpy(f + 26, &src, 4);
    const uint32_t dst = key(8, 8, 8, 8);
    memcpy(f + 30, &dst, 4);
    f[34] = (uint8_t)(sport >> 8), f[35] = (uint8_t)sport, f[36] = 0, f[37] = 53, f[39] = 30;
}

static uint64_t count_of(bng_ctx *c, const char *map) {
    bng_map_info mi{};
    return bng_map_get_info(c, bng_map_id(c, map), &mi) == 0 ? mi.count : ~0ull;
}

static std::shared_ptr<nat::Manager> nat_manager(std::shared_ptr<Backend> be) {
    nat::ManagerConfig cfg;
    cfg.Interface = "eth0";
    cfg.EnableEIM = true;
    cfg.PortsPerSubscriber = 1024;
    cfg.Backend_ = be;
    auto m = *nat::Manager::NewManager(cfg).value;
    CHECK_EQ((bool)m->Start(), false);
    CHECK_EQ((bool)m->AddPublicIP(IPv4(203, 0, 113, 1)), false);
    return m;
}

// two shards; one subscriber per shard with two flows each, flushed through the router with an unknown address
static void test_gpu_two_shards() {
    bng_open_opts o{};
    o.struct_size = sizeof(o), o.device = -1, o.max_batch = 1 << 10, o.max_subscribers = 1 << 10;
    o.max_nat_sessions = 1 << 12, o.max_eim_mappings = 1 << 12, o.event_capacity = 1 << 10, o.world = 2;
    auto dir = std::make_shared<shard::Directory>(2);
    std::vector<std::shared_ptr<Backend>> shards;
    std::vector<std::shared_ptr<nat::Manager>> mgr;
    for (uint32_t i = 0; i < 2; i++) {
        o.rank = i;
        auto b = Backend::Open(&o);
        if (!b->ctx) {
            fprintf(stderr, "FAIL bng_open: %s\n", b->open_error.c_str());
            g_fail++;
            return;
        }
        b->wire_order_keys = true; // addresses as the programs read them off the wire
        shards.push_back(b);
        mgr.push_back(nat_manager(b));
    }
    shard::Router r(shards, dir);
    // a subscriber owned by each shard
    uint32_t ip[2] = {0, 0};
    IP pip[2];
    for (uint32_t s = 0, found = 0; found < 3; s++) {
        const uint32_t k = bng_shard_of_mac(mac_of(s), 2);
        if (found & (1u << k)) continue;
        found |= 1u << k;
        pip[k] = IPv4(10, 7, 0, (uint8_t)(s + 1));
        ip[k] = key(10, 7, 0, (uint8_t)(s + 1));
        dir->Learn(mac_of(s), ip[k]);
    }
    const int prog = bng_prog_id(shards[0]->ctx, "nat44_egress");
    for (uint32_t k = 0; k < 2; k++) {
        CHECK_EQ(mgr[k]->AllocateNAT(pip[k]).ok(), true);
        uint8_t frames[128];
        udp_frame(frames, ip[k], 40000);
        udp_frame(frames + 64, ip[k], 40001);
        uint32_t len[2] = {64, 64};
        uint8_t verdict[2] = {0xff, 0xff};
        bng_batch bt{};
        bt.pkts = frames, bt.len = len, bt.verdict = verdict, bt.n = 2, bt.stride = 64, bt.mem = BNG_MEM_HOST, bt.arena_bytes = 8;
        bt.now_ns = 1000000000ull;
        CHECK_EQ(bng_prog_run(shards[k]->ctx, prog, &bt), 0);
        CHECK_EQ(count_of(shards[k]->ctx, "nat_sessions"), 2ull);
        CHECK_EQ(count_of(shards[k]->ctx, "nat_reverse"), 2ull);
        CHECK_EQ(count_of(shards[k]->ctx, "eim_table"), 2ull);
    }
    const uint32_t addrs[3] = {ip[0], key(192, 0, 2, 1), ip[1]};
    uint64_t rm[3] = {9, 9, 9};
    CHECK_EQ(r.NatFlush(addrs, 3, 2000000000ull, rm), 0);
    CHECK_EQ(rm[0], 4ull);
    CHECK_EQ(rm[1], 4ull);
    CHECK_EQ(rm[2], 4ull);
    for (uint32_t k = 0; k < 2; k++) {
        for (const char *m : {"nat_sessions", "nat_reverse", "eim_table"}) CHECK_EQ(count_of(shards[k]->ctx, m), 0ull);
        CHECK_EQ(count_of(shards[k]->ctx, "subscriber_nat"), 1ull); // the allocation stays: DeallocateNAT removes it
        CHECK_EQ(mgr[k]->DrainLog().size(), (size_t)(2 + 2)); // two SESSION_CREATE, two SESSION_DELETE
    }
    // the manager's flush on one context: nothing left, nothing removed
    uint64_t rm2[3] = {9, 9, 9};
    CHECK_EQ((bool)mgr[0]->FlushSessions({pip[0]}, 3000000000ull, rm2), false);
    CHECK_EQ(rm2[0] + rm2[1] + rm2[2], 0ull);
    CHECK_EQ((bool)mgr[0]->FlushSessions({IP{1, 2, 3}}, 3000000000ull), true); // not an IPv4 address
    CHECK_EQ((bool)mgr[0]->DeallocateNAT(pip[0]), false);
    CHECK_EQ(count_of(shards[0]->ctx, "subscriber_nat"), 0ull);
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    test_grouping();
    if (mode == "gpu") test_gpu_two_shards();
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
