// Tests of the host side of dual-stack attribution: intercept::ParseCC on IPv6 records, the Directory's prefix table
// and longest-prefix steering, and the routing of subscriber_ipv6 by value (bng_host.hpp, bng_shard.hpp).
// `test_dualstack_host cpu` needs no device.  `test_dualstack_host gpu` also installs prefixes through shard::Router,
// moves a subscriber with its prefixes (Router::Move), and checks that 2- and 8-shard runs whose IPv6 frames are
// steered by SteerUpstream / SteerDownstream give the records of one unsharded context.
#include <cstdio>
#include <random>
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

static uint32_t key(uint8_t a, uint8_t b, uint8_t c, uint8_t d) {
    const uint8_t k[4] = {a, b, c, d};
    uint32_t v;
    memcpy(&v, k, 4);
    return v;
}
static uint64_t mac_of(uint32_t s) { return 0x020000000000ull + s * 0x10001ull; }
static uint32_t ip_of(uint32_t s) { return key(100, 64, (uint8_t)(s >> 8), (uint8_t)s); }

// 2001:db8:0:<s>::/64 (kind 0) and the delegated 2001:db9:<s>::/56 (kind 1)
static std::array<uint8_t, 16> prefix(uint32_t s, int kind) {
    std::array<uint8_t, 16> a{};
    a[0] = 0x20, a[1] = 0x01, a[2] = 0x0d, a[3] = kind ? 0xb9 : 0xb8;
    if (kind) a[4] = (uint8_t)(s >> 8), a[5] = (uint8_t)s;
    else a[6] = (uint8_t)(s >> 8), a[7] = (uint8_t)s;
    return a;
}
static bng_ipv6_prefix_key pkey(const std::array<uint8_t, 16> &a, uint32_t plen) { return dualstack::PrefixKey(a.data(), plen); }

// ---------------------------------------------------------------------------
// ParseCC on IPv6 records
// ---------------------------------------------------------------------------
static std::vector<uint8_t> record(const std::vector<uint8_t> &frame, uint32_t cap_len, uint8_t dir) {
    std::vector<uint8_t> r(sizeof(bng_li_record) + frame.size(), 0);
    bng_li_record h{};
    h.cap_len = cap_len, h.wire_len = (uint32_t)frame.size(), h.dir = dir, h.target_id = 7;
    memcpy(r.data(), &h, sizeof(h));
    memcpy(r.data() + sizeof(h), frame.data(), frame.size());
    return r;
}
static std::vector<uint8_t> v6frame(uint8_t next, const std::vector<uint8_t> &l4) {
    std::vector<uint8_t> f(54 + l4.size(), 0);
    f[12] = 0x86, f[13] = 0xDD, f[14] = 0x60, f[20] = next, f[21] = 64;
    for (int i = 0; i < 16; i++) f[22 + i] = (uint8_t)(0x10 + i), f[38 + i] = (uint8_t)(0x80 + i);
    std::copy(l4.begin(), l4.end(), f.begin() + 54);
    return f;
}
static void test_parse_cc() {
    using intercept::CC;
    const IP src(16, 0), dst(16, 0);
    IP s6, d6;
    for (int i = 0; i < 16; i++) s6.push_back((uint8_t)(0x10 + i)), d6.push_back((uint8_t)(0x80 + i));
    CC cc;
    { // TCP uplink
        auto f = v6frame(6, {0x1f, 0x90, 0x00, 0x50, 1, 2, 3, 4});
        auto r = record(f, (uint32_t)f.size(), BNG_LI_UPLINK);
        CHECK(intercept::ParseCC(r.data(), &cc));
        CHECK(cc.src == s6 && cc.dst == d6 && cc.protocol == 6 && cc.src_port == 8080 && cc.dst_port == 80);
        CHECK(cc.payload.size() == f.size() - 14 && cc.rec.target_id == 7);
    }
    { // UDP downlink
        auto f = v6frame(17, {0x13, 0x88, 0x00, 0x35, 0, 8, 0, 0});
        auto r = record(f, (uint32_t)f.size(), BNG_LI_DOWNLINK);
        CHECK(intercept::ParseCC(r.data(), &cc));
        CHECK(cc.direction == intercept::Direction::Downlink && cc.protocol == 17 && cc.src_port == 5000 && cc.dst_port == 53);
    }
    { // ICMPv6 echo request uplink / echo reply downlink: the echo id as the subscriber-side port; other types: none
        auto f = v6frame(58, {128, 0, 0, 0, 0x12, 0x34, 0, 1});
        auto r = record(f, (uint32_t)f.size(), BNG_LI_UPLINK);
        CHECK(intercept::ParseCC(r.data(), &cc));
        CHECK(cc.protocol == 58 && cc.src_port == 0x1234 && cc.dst_port == 0);
        f = v6frame(58, {129, 0, 0, 0, 0x43, 0x21, 0, 1});
        r = record(f, (uint32_t)f.size(), BNG_LI_DOWNLINK);
        CHECK(intercept::ParseCC(r.data(), &cc));
        CHECK(cc.src_port == 0 && cc.dst_port == 0x4321);
        f = v6frame(58, {1, 4, 0, 0, 0x43, 0x21, 0, 1});
        r = record(f, (uint32_t)f.size(), BNG_LI_DOWNLINK);
        CHECK(intercept::ParseCC(r.data(), &cc));
        CHECK(cc.src_port == 0 && cc.dst_port == 0);
    }
    { // behind an extension header (hop-by-hop, then TCP): the next header as the protocol, ports 0
        auto f = v6frame(0, {6, 0, 1, 0, 0, 0, 0, 0, 0x1f, 0x90, 0x00, 0x50});
        auto r = record(f, (uint32_t)f.size(), BNG_LI_UPLINK);
        CHECK(intercept::ParseCC(r.data(), &cc));
        CHECK(cc.protocol == 0 && cc.src_port == 0 && cc.dst_port == 0 && cc.src == s6);
    }
    { // short captures
        auto f = v6frame(6, {0x1f, 0x90, 0x00, 0x50});
        auto r = record(f, 56, BNG_LI_UPLINK); // addresses, not the ports
        CHECK(intercept::ParseCC(r.data(), &cc));
        CHECK(cc.src == s6 && cc.dst == d6 && cc.src_port == 0 && cc.dst_port == 0);
        r = record(f, 40, BNG_LI_UPLINK); // the source, not the destination
        CHECK(!intercept::ParseCC(r.data(), &cc));
        CHECK(cc.src == s6 && cc.dst == dst && cc.protocol == 6 && cc.payload.size() == 26);
        r = record(f, 30, BNG_LI_UPLINK);
        CHECK(!intercept::ParseCC(r.data(), &cc));
        CHECK(cc.src == src && cc.dst == dst);
        r = record(f, 10, BNG_LI_UPLINK); // not even the ethertype: parsed as IPv4, nothing there
        CHECK(!intercept::ParseCC(r.data(), &cc));
        CHECK(cc.src == IPv4(0, 0, 0, 0) && cc.payload.empty());
    }
    { // IPv4 is parsed as before
        std::vector<uint8_t> f(42, 0);
        f[12] = 0x08, f[14] = 0x45, f[23] = 17;
        f[26] = 100, f[27] = 64, f[28] = 0, f[29] = 10, f[30] = 8, f[31] = 8, f[32] = 4, f[33] = 4;
        f[34] = 0x1f, f[35] = 0x90, f[36] = 0, f[37] = 53;
        auto r = record(f, 42, BNG_LI_UPLINK);
        CHECK(intercept::ParseCC(r.data(), &cc));
        CHECK(cc.src == IPv4(100, 64, 0, 10) && cc.dst == IPv4(8, 8, 4, 4) && cc.src_port == 8080 && cc.dst_port == 53);
    }
}

// ---------------------------------------------------------------------------
// Directory: prefixes, longest match, steering; Router: routing by value
// ---------------------------------------------------------------------------
static std::vector<uint8_t> down6(const std::array<uint8_t, 16> &dst, uint8_t host) {
    std::vector<uint8_t> f(64, 0);
    f[12] = 0x86, f[13] = 0xDD, f[14] = 0x60, f[20] = 17;
    memcpy(f.data() + 38, dst.data(), 16);
    f[53] = host;
    return f;
}
static void test_directory() {
    for (uint32_t world : {2u, 8u}) {
        auto dir = std::make_shared<shard::Directory>(world);
        for (uint32_t s = 0; s < 64; s++) dir->Learn(mac_of(s), ip_of(s));
        // sub 0: 2001:db9:0::/56; sub 1: a /60 inside it; sub 2: a /128 inside that
        auto p56 = prefix(0, 1), p60 = p56, p128 = p56;
        p60[7] = 0x10; // bits 56-59
        p128[7] = 0x10, p128[15] = 9;
        CHECK(dir->LearnPrefix(p56.data(), 56, ip_of(0)));
        CHECK(dir->LearnPrefix(p60.data(), 60, ip_of(1)));
        CHECK(dir->LearnPrefix(p128.data(), 128, ip_of(2)));
        CHECK(!dir->LearnPrefix(p56.data(), 129, ip_of(3)));
        auto a = p128;
        CHECK(*dir->OwnerOfV6(a.data()) == ip_of(2));
        CHECK(*dir->OwnerOfV6(a.data(), 127) == ip_of(1));
        CHECK(*dir->OwnerOfV6(a.data(), 59) == ip_of(0));
        a[15] = 10;
        CHECK(*dir->OwnerOfV6(a.data()) == ip_of(1));
        a[7] = 0x20;
        CHECK(*dir->OwnerOfV6(a.data()) == ip_of(0));
        a[5] = 1; // outside every prefix
        CHECK(!dir->OwnerOfV6(a.data()));
        // a key with bits past prefixlen set is the same prefix
        auto noisy = p56;
        noisy[7] = 0xAB, noisy[15] = 0xCD;
        CHECK(*dir->PrefixOwner(noisy.data(), 56) == ip_of(0));
        // steering: the destination's owner; no owner, tagged, short and IPv4-without-a-block frames: fallback
        for (uint8_t h : {1, 9, 200}) {
            auto f = down6(p60, h);
            f[52] = h == 9 ? 0 : 7;
            auto want = dir->ShardOfIP(*dir->OwnerOfV6(f.data() + 38));
            CHECK(dir->SteerDownstream(f.data(), 64, 99) == *want);
        }
        auto out = down6(a, 1);
        CHECK(dir->SteerDownstream(out.data(), 64, 99) == 99u);
        auto f = down6(p56, 1);
        CHECK(dir->SteerDownstream(f.data(), 53, 99) == 99u);
        f[12] = 0x81, f[13] = 0x00;
        CHECK(dir->SteerDownstream(f.data(), 64, 99) == 99u);
        dir->ForgetPrefix(p128.data(), 128);
        CHECK(*dir->OwnerOfV6(p128.data()) == ip_of(1));
        // routing by value
        CHECK(shard::RouteOf("subscriber_ipv6") == shard::Route::ByValueIP);
        std::vector<std::shared_ptr<Backend>> shards;
        for (uint32_t i = 0; i < world; i++) shards.push_back(std::make_shared<Backend>()); // never opened
        shard::Router r(shards, dir);
        for (uint32_t s = 0; s < 64; s++) {
            auto k = pkey(prefix(s, 0), 64);
            const uint32_t v = ip_of(s);
            CHECK(r.Owner("subscriber_ipv6", &k, &v) == (int)dir->ShardOfMAC(mac_of(s)));
        }
        auto k = pkey(p60, 60);
        CHECK(r.Owner("subscriber_ipv6", &k) == (int)dir->ShardOfMAC(mac_of(1))); // without the value: as learned
        const uint32_t unknown = key(10, 9, 9, 9);
        CHECK(r.Owner("subscriber_ipv6", &k, &unknown) == -ENOENT);
        k.prefixlen = 129;
        CHECK(r.Owner("subscriber_ipv6", &k, &unknown) == -EINVAL);
        k = pkey(prefix(63, 1), 56);
        CHECK(r.Owner("subscriber_ipv6", &k) == -ENOENT); // never learned
    }
}

// ---------------------------------------------------------------------------
// on the GPU
// ---------------------------------------------------------------------------
static uint64_t count_of(bng_ctx *c, const char *map) {
    bng_map_info mi{};
    return bng_map_get_info(c, bng_map_id(c, map), &mi) == 0 ? mi.count : ~0ull;
}
static std::shared_ptr<Backend> open_shard(uint32_t rank, uint32_t world) {
    bng_open_opts o{};
    o.struct_size = sizeof(o), o.device = -1, o.max_batch = 1 << 14, o.max_subscribers = 1 << 10;
    o.max_nat_sessions = 1 << 10, o.max_eim_mappings = 1 << 10, o.event_capacity = 1 << 10, o.world = world, o.rank = rank;
    auto b = Backend::Open(&o);
    if (!b->ctx) {
        fprintf(stderr, "FAIL bng_open: %s\n", b->open_error.c_str());
        g_fail++;
    }
    return b;
}
// a subscriber: its directory entry (an unlimited qos_ingress bucket) on its owner shard, and its two prefixes
static void provision(shard::Router &r, uint32_t s) {
    r.Dir().Learn(mac_of(s), ip_of(s));
    const uint32_t ip = ip_of(s);
    uint8_t tb[32] = {};
    CHECK(r.Update("qos_ingress", &ip, tb) == 0);
    for (int kind = 0; kind < 2; kind++) {
        auto k = pkey(prefix(s, kind), kind ? 56 : 64);
        CHECK(r.Update("subscriber_ipv6", &k, &ip) == 0);
    }
}
static void run(bng_ctx *c, const char *prog, std::vector<uint8_t> &frames) {
    const uint32_t n = (uint32_t)(frames.size() / 64);
    if (!n) return;
    std::vector<uint32_t> len(n, 64);
    std::vector<uint8_t> verdict(n);
    bng_batch bt{};
    bt.pkts = frames.data(), bt.len = len.data(), bt.verdict = verdict.data(), bt.n = n, bt.stride = 64;
    bt.mem = BNG_MEM_HOST, bt.arena_bytes = (uint32_t)(frames.size() / 16), bt.now_ns = 1000000000ull;
    CHECK(bng_prog_run(c, bng_prog_id(c, prog), &bt) == 0);
}

static void test_gpu_routes_and_move() {
    auto dir = std::make_shared<shard::Directory>(2);
    std::vector<std::shared_ptr<Backend>> shards = {open_shard(0, 2), open_shard(1, 2)};
    if (!shards[0]->ctx || !shards[1]->ctx) return;
    shard::Router r(shards, dir);
    uint64_t on[2] = {0, 0};
    for (uint32_t s = 0; s < 16; s++) provision(r, s), on[dir->ShardOfMAC(mac_of(s))] += 2;
    for (size_t k = 0; k < 2; k++) CHECK(count_of(shards[k]->ctx, "subscriber_ipv6") == on[k]); // on the owner only
    // the router's lookup is the longest match on the owner's shard
    auto a = prefix(5, 1);
    a[15] = 1;
    auto k = pkey(a, 128);
    uint32_t v = 0;
    CHECK(r.Lookup("subscriber_ipv6", &k, &v) == 0 && v == ip_of(5));
    // a prefix handed to a subscriber on the other shard leaves its old shard
    uint32_t s2 = 1;
    while (dir->ShardOfMAC(mac_of(s2)) == dir->ShardOfMAC(mac_of(0))) s2++;
    k = pkey(prefix(0, 1), 56);
    const uint32_t ip2 = ip_of(s2);
    CHECK(r.Update("subscriber_ipv6", &k, &ip2) == 0);
    const size_t sh0 = dir->ShardOfMAC(mac_of(0)), sh2 = dir->ShardOfMAC(mac_of(s2));
    CHECK(count_of(shards[sh0]->ctx, "subscriber_ipv6") == on[sh0] - 1);
    CHECK(count_of(shards[sh2]->ctx, "subscriber_ipv6") == on[sh2] + 1);
    on[sh0]--, on[sh2]++;
    CHECK(r.Delete("subscriber_ipv6", &k) == 0);
    on[sh2]--;
    CHECK(count_of(shards[sh2]->ctx, "subscriber_ipv6") == on[sh2]);
    CHECK(!dir->PrefixOwner(k.addr, 56));
    CHECK(r.Delete("subscriber_ipv6", &k) == -ENOENT);
    // Router::Move carries the subscriber's prefixes, and downstream IPv6 steering follows
    const uint32_t s = 3;
    const size_t from = dir->ShardOfMAC(mac_of(s)), to = 1 - from;
    CHECK(r.Move(from, to, {ip_of(s)}, {mac_of(s)}) == 0);
    CHECK(count_of(shards[from]->ctx, "subscriber_ipv6") == on[from] - 2);
    CHECK(count_of(shards[to]->ctx, "subscriber_ipv6") == on[to] + 2);
    auto f = down6(prefix(s, 0), 5);
    CHECK(dir->SteerDownstream(f.data(), 64, 99) == (uint32_t)to);
    k = pkey(prefix(s, 0), 64);
    v = 0;
    CHECK(r.Lookup("subscriber_ipv6", &k, &v) == 0 && v == ip_of(s));
}

// 2 / 8 shards against one context: IPv6 frames steered by SteerUpstream (source MAC) and SteerDownstream (destination
// prefix) give every subscriber the record the unsharded run gives it, and no other shard holds a count
static void test_gpu_sharded_union(uint32_t world) {
    const uint32_t nsub = 48;
    auto one = open_shard(0, 1);
    if (!one->ctx) return;
    auto dir1 = std::make_shared<shard::Directory>(1);
    shard::Router r1({one}, dir1);
    auto dir = std::make_shared<shard::Directory>(world);
    std::vector<std::shared_ptr<Backend>> shards;
    for (uint32_t i = 0; i < world; i++) shards.push_back(open_shard(i, world));
    for (auto &b : shards)
        if (!b->ctx) return;
    shard::Router r(shards, dir);
    for (uint32_t s = 0; s < nsub; s++) provision(r, s), provision(r1, s);
    std::vector<std::shared_ptr<Backend>> all = shards;
    all.push_back(one);
    for (auto &b : all) {
        CHECK(bng_acct_enable(b->ctx, bng_prog_id(b->ctx, "qos_ingress_prog"), 1) == 0);
        CHECK(bng_acct_enable(b->ctx, bng_prog_id(b->ctx, "qos_egress_prog"), 1) == 0);
    }
    std::mt19937 rng(world);
    std::vector<uint8_t> up1, down1;
    std::vector<std::vector<uint8_t>> up(world), down(world);
    for (int i = 0; i < 3000; i++) {
        const uint32_t s = rng() % nsub;
        auto a = prefix(rng() % 8 == 0 ? nsub + 5 : s, (int)(rng() & 1)); // some addresses no prefix covers
        for (int j = 8; j < 16; j++) a[j] = (uint8_t)rng();
        const bool is_down = rng() & 1;
        std::vector<uint8_t> f(64, 0);
        uint8_t m[6];
        uint64_t mac = mac_of(s);
        for (int j = 5; j >= 0; j--) m[j] = (uint8_t)mac, mac >>= 8;
        memcpy(f.data() + (is_down ? 0 : 6), m, 6);
        f[12] = 0x86, f[13] = 0xDD, f[14] = 0x60, f[20] = 17;
        memcpy(f.data() + (is_down ? 38 : 22), a.data(), 16);
        const uint32_t k = is_down ? dir->SteerDownstream(f.data(), 64, 0) : dir->SteerUpstream(f.data(), 64);
        auto &dst = is_down ? down[k] : up[k];
        dst.insert(dst.end(), f.begin(), f.end());
        (is_down ? down1 : up1).insert((is_down ? down1 : up1).end(), f.begin(), f.end());
    }
    run(one->ctx, "qos_ingress_prog", up1);
    run(one->ctx, "qos_egress_prog", down1);
    for (uint32_t k = 0; k < world; k++) {
        run(shards[k]->ctx, "qos_ingress_prog", up[k]);
        run(shards[k]->ctx, "qos_egress_prog", down[k]);
    }
    uint64_t total = 0, bad = 0;
    for (uint32_t s = 0; s < nsub; s++) {
        uint32_t ip = ip_of(s);
        bng_acct want{}, got{};
        int32_t res = 0;
        CHECK(bng_acct_read(one->ctx, &ip, 1, &want, &res) == 0 && res == 0);
        CHECK(r.AcctRead(ip, &got) == 0);
        bad += memcmp(&want, &got, sizeof(want)) != 0;
        total += want.up_packets + want.down_packets;
    }
    CHECK(bad == 0);
    CHECK(total > 2000);
    uint64_t sum = 0; // no record anywhere but on the owner
    for (uint32_t k = 0; k < world; k++) {
        std::vector<uint32_t> addrs(2048);
        std::vector<bng_acct> recs(2048);
        int64_t n = bng_acct_dump(shards[k]->ctx, addrs.data(), recs.data(), 2048);
        for (int64_t i = 0; i < n; i++) sum += recs[i].up_packets + recs[i].down_packets;
    }
    CHECK(sum == total);
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    test_parse_cc();
    test_directory();
    if (mode == "gpu") {
        test_gpu_routes_and_move();
        test_gpu_sharded_union(2);
        test_gpu_sharded_union(8);
    }
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
