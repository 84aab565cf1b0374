// Tests of the host side of the subscriber hand-over (bng_shard.hpp): with no pins every route of Directory / Router
// is bng_shard_of_mac's; a pin redirects every route; Drain's destinations.  `test_move_host cpu` needs no device;
// `test_move_host gpu` also moves subscribers with flows between two dataplane contexts through Router::Move and
// Router::Drain, including the rollback of an import the destination refuses.
#include <cstdio>
#include <random>
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

static void mac_bytes(uint64_t mac, uint8_t *m) { // MacKey's inverse
    for (int i = 5; i >= 0; i--) m[i] = (uint8_t)mac, mac >>= 8;
}

// An inbound UDP frame to (public key, port).
static void down_frame(uint8_t *f, uint32_t pub, uint16_t port) {
    memset(f, 0, 64);
    f[12] = 0x08, f[14] = 0x45, f[23] = 17;
    memcpy(f + 30, &pub, 4);
    f[36] = (uint8_t)(port >> 8), f[37] = (uint8_t)port;
}

// With no pins, every route is what it was before pins existed: bng_shard_of_mac of the subscriber's MAC.
static void test_no_pins() {
    std::mt19937_64 rng(7);
    for (uint32_t world : {2u, 3u, 8u}) {
        auto dir = std::make_shared<shard::Directory>(world);
        std::vector<std::shared_ptr<Backend>> shards;
        for (uint32_t i = 0; i < world; i++) shards.push_back(std::make_shared<Backend>()); // never opened
        shard::Router r(shards, dir);
        const uint32_t pub = key(203, 0, 113, 9);
        uint64_t bad = 0;
        for (uint32_t s = 0; s < 100000; s++) {
            const uint64_t mac = rng() & 0xFFFFFFFFFFFFull;
            const uint32_t ip = (uint32_t)rng();
            dir->Learn(mac, ip);
            const uint32_t want = bng_shard_of_mac(mac, world);
            bad += dir->ShardOfMAC(mac) != want;
            auto si = dir->ShardOfIP(ip);
            bad += !si || *si != want;
            uint8_t m[8];
            mac_bytes(mac, m);
            uint8_t f[64] = {};
            memcpy(f + 6, m, 6);
            bad += dir->SteerUpstream(f, 64) != want;
            bad += r.Owner("subscriber_bindings", &mac) != (int)want;
            bad += r.Owner("subscriber_nat", &ip) != (int)want;
            if (s < 60) { // 60 blocks of 1024 ports from 1024 on
                const uint16_t start = (uint16_t)(1024 + s * 1024);
                dir->AddBlock(pub, start, ip);
                auto sp = dir->ShardOfPublic(pub, (uint16_t)(start + 5));
                bad += !sp || *sp != want;
                down_frame(f, pub, (uint16_t)(start + 5));
                bad += dir->SteerDownstream(f, 64, 99) != want;
            }
        }
        CHECK_EQ(bad, 0ull);
    }
}

static void test_pins() {
    const uint32_t world = 4;
    shard::Directory dir(world);
    const uint64_t mac = mac_of(3);
    const uint32_t ip = key(10, 0, 0, 3), pub = key(203, 0, 113, 1);
    dir.Learn(mac, ip);
    dir.AddBlock(pub, 2048, ip);
    const uint32_t home = bng_shard_of_mac(mac, world), other = (home + 1) % world;
    uint8_t up[64] = {}, dn[64];
    mac_bytes(mac, up + 6);
    down_frame(dn, pub, 2050);
    dir.Pin(mac, other);
    CHECK_EQ(dir.ShardOfMAC(mac), other);
    CHECK_EQ(*dir.ShardOfIP(ip), other);
    CHECK_EQ(*dir.ShardOfPublic(pub, 2050), other);
    CHECK_EQ(dir.SteerUpstream(up, 64), other);
    CHECK_EQ(dir.SteerDownstream(dn, 64, 99), other);
    CHECK_EQ(dir.ShardOfMAC(mac_of(4)), bng_shard_of_mac(mac_of(4), world)); // other MACs keep their hash
    dir.Unpin(mac);
    CHECK_EQ(dir.ShardOfMAC(mac), home);
    CHECK_EQ(*dir.ShardOfIP(ip), home);
    CHECK_EQ(dir.SteerDownstream(dn, 64, 99), home);
    // Forget drops the pin: a returning MAC is placed by the hash again
    dir.Pin(mac, other);
    dir.Forget(mac);
    CHECK_EQ(dir.ShardOfMAC(mac), home);
    CHECK_EQ(dir.ShardOfIP(ip).has_value(), false);
    // a CPE swap: the address learned for a new MAC, then the old MAC forgotten, in either order
    for (int order = 0; order < 2; order++) {
        uint64_t nmac = mac_of(100);
        while (bng_shard_of_mac(nmac, world) == home) nmac++;
        dir.Learn(mac, ip);
        if (order) dir.Forget(mac);
        dir.Learn(nmac, ip);
        if (!order) dir.Forget(mac);
        CHECK_EQ(*dir.ShardOfIP(ip), bng_shard_of_mac(nmac, world));
        CHECK_EQ(dir.SubscribersOn(home).size(), (size_t)0);
        dir.Forget(nmac);
    }
}

// Drain(k)'s destinations: never k, always a shard, the same every time, and spread over the other shards.
static void test_drain_targets() {
    for (uint32_t world : {2u, 3u, 8u}) {
        auto dir = std::make_shared<shard::Directory>(world);
        std::vector<std::shared_ptr<Backend>> shards;
        for (uint32_t i = 0; i < world; i++) shards.push_back(std::make_shared<Backend>());
        shard::Router r(shards, dir);
        for (uint32_t s = 0; s < 4000; s++) dir->Learn(mac_of(s), key(10, 2, (uint8_t)(s >> 8), (uint8_t)s));
        for (uint32_t k = 0; k < world; k++) {
            std::vector<uint64_t> per(world, 0);
            uint64_t bad = 0;
            for (const auto &e : dir->SubscribersOn(k)) {
                bad += dir->ShardOfMAC(e.first) != k;
                const size_t t = r.DrainTarget(k, e.first);
                bad += t == k || t >= world || t != r.DrainTarget(k, e.first);
                if (t < world) per[t]++;
            }
            CHECK_EQ(bad, 0ull);
            for (uint32_t t = 0; t < world; t++)
                if (t != k) CHECK_EQ(per[t] > 0, true);
        }
        CHECK_EQ(r.Drain(world), -EINVAL);
    }
    shard::Router one({std::make_shared<Backend>()}, std::make_shared<shard::Directory>(1));
    CHECK_EQ(one.Drain(0), -EINVAL); // nowhere to go
}

// ---- on real contexts ----
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

static std::shared_ptr<Backend> open_shard(uint32_t rank, uint32_t max_sess) {
    bng_open_opts o{};
    o.struct_size = sizeof(o), o.device = -1, o.max_batch = 1 << 10, o.max_subscribers = 1 << 10;
    o.max_nat_sessions = max_sess, o.max_eim_mappings = 1 << 12, o.event_capacity = 1 << 10, o.world = 2, o.rank = rank;
    auto b = Backend::Open(&o);
    if (!b->ctx) {
        fprintf(stderr, "FAIL bng_open: %s\n", b->open_error.c_str());
        g_fail++;
    }
    return b;
}

// one NAT manager per shard, each with a public address of its own (so that no two shards hold the same reverse key)
static std::shared_ptr<nat::Manager> nat_manager(std::shared_ptr<Backend> be, uint8_t pub) {
    nat::ManagerConfig cfg;
    cfg.Interface = "eth0";
    cfg.EnableEIM = true;
    cfg.PortsPerSubscriber = 1024;
    cfg.Backend_ = be;
    auto m = *nat::Manager::NewManager(cfg).value;
    CHECK_EQ((bool)m->Start(), false);
    CHECK_EQ((bool)m->AddPublicIP(IPv4(203, 0, 113, pub)), false);
    return m;
}

// subscriber s: a NAT block from its owner's manager, a subscriber_bindings entry and two upstream flows on its owner
static uint32_t provision(shard::Router &r, std::vector<std::shared_ptr<nat::Manager>> &mgr, uint32_t s) {
    const uint32_t ip = key(10, 7, 0, (uint8_t)(s + 1));
    const uint64_t mac = mac_of(s);
    r.Dir().Learn(mac, ip);
    const size_t k = r.Dir().ShardOfMAC(mac);
    CHECK_EQ(mgr[k]->AllocateNAT(IPv4(10, 7, 0, (uint8_t)(s + 1))).ok(), true);
    uint8_t binding[24] = {};
    CHECK_EQ(r.Update("subscriber_bindings", &mac, binding), 0);
    bng_ctx *c = r.Shard(k).ctx;
    uint8_t frames[128];
    udp_frame(frames, ip, 40000);
    udp_frame(frames + 64, ip, 40001);
    uint32_t len[2] = {64, 64};
    uint8_t verdict[2] = {0xff, 0xff};
    bng_batch bt{};
    bt.pkts = frames, bt.len = len, bt.verdict = verdict, bt.n = 2, bt.stride = 64, bt.mem = BNG_MEM_HOST, bt.arena_bytes = 8;
    bt.now_ns = 1000000000ull;
    CHECK_EQ(bng_prog_run(c, bng_prog_id(c, "nat44_egress"), &bt), 0);
    return ip;
}

static void test_gpu_move() {
    const char *flow[3] = {"nat_sessions", "nat_reverse", "eim_table"};
    { // Move and Drain between two shards
        auto dir = std::make_shared<shard::Directory>(2);
        std::vector<std::shared_ptr<Backend>> shards = {open_shard(0, 1 << 12), open_shard(1, 1 << 12)};
        if (!shards[0]->ctx || !shards[1]->ctx) return;
        for (auto &b : shards) b->wire_order_keys = true;
        shard::Router r(shards, dir);
        std::vector<std::shared_ptr<nat::Manager>> mgr = {nat_manager(shards[0], 1), nat_manager(shards[1], 2)};
        std::vector<uint32_t> ip(8);
        uint64_t on[2] = {0, 0};
        for (uint32_t s = 0; s < 8; s++) ip[s] = provision(r, mgr, s), on[dir->ShardOfMAC(mac_of(s))]++;
        for (size_t k = 0; k < 2; k++) CHECK_EQ(count_of(shards[k]->ctx, "nat_sessions"), 2 * on[k]);
        // move subscriber 0 to the other shard
        const size_t from = dir->ShardOfMAC(mac_of(0)), to = 1 - from;
        CHECK_EQ(r.Move(from, to, {ip[0]}, {mac_of(0)}), 0);
        CHECK_EQ(dir->ShardOfMAC(mac_of(0)), (uint32_t)to);
        CHECK_EQ(*dir->ShardOfIP(ip[0]), (uint32_t)to);
        on[from]--, on[to]++;
        for (size_t k = 0; k < 2; k++) {
            for (const char *m : flow) CHECK_EQ(count_of(shards[k]->ctx, m), 2 * on[k]);
            CHECK_EQ(count_of(shards[k]->ctx, "subscriber_nat"), on[k]);
            CHECK_EQ(count_of(shards[k]->ctx, "subscriber_bindings"), on[k]);
        }
        // drain shard 0: everything ends on shard 1, pinned there
        CHECK_EQ(r.Drain(0), 0);
        for (const char *m : flow) CHECK_EQ(count_of(shards[0]->ctx, m), 0ull);
        for (const char *m : flow) CHECK_EQ(count_of(shards[1]->ctx, m), 16ull);
        CHECK_EQ(count_of(shards[0]->ctx, "subscriber_nat"), 0ull);
        CHECK_EQ(count_of(shards[1]->ctx, "subscriber_nat"), 8ull);
        CHECK_EQ(dir->SubscribersOn(0).size(), (size_t)0);
        for (uint32_t s = 0; s < 8; s++) CHECK_EQ(r.Owner("subscriber_nat", &ip[s]), 1);
    }
    { // rollback: the destination has room for one session only
        auto dir = std::make_shared<shard::Directory>(2);
        std::vector<std::shared_ptr<Backend>> shards = {open_shard(0, 1 << 12), open_shard(1, 1)};
        if (!shards[0]->ctx || !shards[1]->ctx) return;
        for (auto &b : shards) b->wire_order_keys = true;
        shard::Router r(shards, dir);
        std::vector<std::shared_ptr<nat::Manager>> mgr = {nat_manager(shards[0], 1), nat_manager(shards[1], 2)};
        uint32_t s = 0;
        while (dir->ShardOfMAC(mac_of(s)) != 0) s++;
        const uint32_t ip = provision(r, mgr, s);
        bng_ctx *c0 = shards[0]->ctx;
        uint64_t before[3];
        for (int t = 0; t < 3; t++) before[t] = count_of(c0, flow[t]);
        CHECK_EQ(before[0], 2ull);
        CHECK_EQ(r.Move(0, 1, {ip}, {mac_of(s)}), -E2BIG);
        for (int t = 0; t < 3; t++) CHECK_EQ(count_of(c0, flow[t]), before[t]);
        CHECK_EQ(count_of(c0, "subscriber_nat"), 1ull);
        CHECK_EQ(count_of(c0, "subscriber_bindings"), 1ull);
        CHECK_EQ(count_of(shards[1]->ctx, "nat_sessions"), 0ull);
        CHECK_EQ(count_of(shards[1]->ctx, "subscriber_nat"), 0ull);
        CHECK_EQ(dir->ShardOfMAC(mac_of(s)), 0u); // no pin
        CHECK_EQ(r.Drain(0), -E2BIG);
        CHECK_EQ(count_of(c0, "nat_sessions"), 2ull);
    }
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    test_no_pins();
    test_pins();
    test_drain_targets();
    if (mode == "gpu") test_gpu_move();
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
