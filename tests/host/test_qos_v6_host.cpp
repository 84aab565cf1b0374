// Tests of the host side of IPv6 shaping (bng_qos_ipv6_enable): qos::ManagerConfig::ShapeIPv6 applied by
// qos::Manager::Start, and shard::Router::QoSIPv6Enable reaching every shard (bng_host.hpp, bng_shard.hpp).
// `test_qos_v6_host cpu` needs no device: the NULL-context check.  `test_qos_v6_host gpu` observes the flag through
// its effect: a subscriber whose upload bucket holds 64 KiB sends 100 IPv6 frames of 1000 bytes, and exactly those
// past the bucket are dropped when shaping is on, none when it is off.
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

// 2001:db8:0:<s>::/64
static std::array<uint8_t, 16> prefix(uint8_t s) {
    std::array<uint8_t, 16> a{};
    a[0] = 0x20, a[1] = 0x01, a[2] = 0x0d, a[3] = 0xb8, a[7] = s;
    return a;
}

// Subscriber 100.64.0.<s> gets a full 64 KiB upload bucket at 8 kbit/s and the prefix above, then sends 100 IPv6
// frames of 1000 bytes from it through qos_ingress_prog in one batch.  Returns the frames dropped.
static int send_v6(bng_ctx *c, uint8_t s, uint64_t now_ns) {
    const uint8_t ip[4] = {100, 64, 0, s};
    uint32_t key;
    memcpy(&key, ip, 4);
    qos::TokenBucket tb;
    tb.RateBPS = 8000, tb.BurstBytes = 65536, tb.Tokens = 65536, tb.LastUpdate = now_ns;
    CHECK(bng_map_update(c, bng_map_id(c, "qos_ingress"), &key, &tb, BNG_ANY) == 0);
    const auto p = prefix(s);
    CHECK(dualstack::SetPrefix(c, p.data(), 64, key, false) == 0);
    const uint32_t n = 100;
    std::vector<uint8_t> frames(n * 64);
    for (uint32_t i = 0; i < n; i++) {
        uint8_t *f = &frames[i * 64];
        f[12] = 0x86, f[13] = 0xDD, f[14] = 0x60, f[20] = 17, f[21] = 64;
        memcpy(f + 22, p.data(), 16);
        f[37] = (uint8_t)(i + 1);
    }
    std::vector<uint32_t> len(n, 1000);
    std::vector<uint8_t> verdict(n);
    bng_batch bt{};
    bt.pkts = frames.data(), bt.len = len.data(), bt.verdict = verdict.data(), bt.n = n, bt.stride = 64;
    bt.mem = BNG_MEM_HOST, bt.arena_bytes = (uint32_t)(frames.size() / 16), bt.now_ns = now_ns;
    CHECK(bng_prog_run(c, bng_prog_id(c, "qos_ingress_prog"), &bt) == 0);
    int shot = 0;
    for (uint8_t v : verdict) shot += v == BNG_TC_ACT_SHOT;
    return shot;
}
static const int k_dropped = 100 - 65536 / 1000; // what the bucket cannot hold

static void test_null() { CHECK(bng_qos_ipv6_enable(nullptr, 1) == -EINVAL && bng_qos_ipv6_enable(nullptr, 0) == -EINVAL); }

static void test_gpu_manager() {
    for (bool shape : {false, true}) {
        auto be = open_ctx(0, 1);
        if (!be->ctx) return;
        qos::ManagerConfig cfg;
        cfg.Interface = "eth0", cfg.Backend_ = be, cfg.ShapeIPv6 = shape;
        auto m = qos::Manager::NewManager(cfg);
        CHECK(m.ok());
        CHECK(send_v6(be->ctx, 1, 1000000000ull) == 0); // NewManager alone applies nothing
        CHECK(!(*m)->Start());
        CHECK(send_v6(be->ctx, 2, 2000000000ull) == (shape ? k_dropped : 0));
        // SetSubscriberQoS needs nothing new: the IPv4 buckets it writes shape the subscriber's IPv6 frames
        qos::SubscriberQoS q;
        q.Addr = IPv4(100, 64, 0, 2), q.UploadBPS = 8000, q.DownloadBPS = 8000;
        CHECK(!(*m)->SetSubscriberQoS(q));
    }
}

static void test_gpu_router() {
    auto dir = std::make_shared<shard::Directory>(2);
    std::vector<std::shared_ptr<Backend>> shards = {open_ctx(0, 2), open_ctx(1, 2)};
    if (!shards[0]->ctx || !shards[1]->ctx) return;
    shard::Router r(shards, dir);
    uint8_t s = 1;
    uint64_t now = 1000000000ull;
    for (size_t k = 0; k < 2; k++) CHECK(send_v6(shards[k]->ctx, s++, now += 1000000000ull) == 0); // off by default
    CHECK(r.QoSIPv6Enable(true) == 0);
    for (size_t k = 0; k < 2; k++) CHECK(send_v6(shards[k]->ctx, s++, now += 1000000000ull) == k_dropped);
    CHECK(r.QoSIPv6Enable(false) == 0);
    for (size_t k = 0; k < 2; k++) CHECK(send_v6(shards[k]->ctx, s++, now += 1000000000ull) == 0);
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    test_null();
    if (mode == "gpu") {
        test_gpu_manager();
        test_gpu_router();
    }
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
