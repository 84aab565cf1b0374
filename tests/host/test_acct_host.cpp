// Tests of the host side of per-subscriber accounting: the RADIUS counter source (bng_host.hpp, radius::) and the
// routing of a read to the owner shard (bng_shard.hpp, Router::AcctRead).
// `test_acct_host cpu` needs no device; `test_acct_host gpu` also counts one frame on a dataplane context and reads
// it back through the counter source.
#include <cstddef>
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

static void test_layout() {
    CHECK_EQ(sizeof(bng_acct), (size_t)64);
    CHECK_EQ(offsetof(bng_acct, up_bytes), (size_t)8);
    CHECK_EQ(offsetof(bng_acct, up_drop_packets), (size_t)16);
    CHECK_EQ(offsetof(bng_acct, down_packets), (size_t)32);
    CHECK_EQ(offsetof(bng_acct, down_drop_bytes), (size_t)56);
}

static void test_counter_mapping() {
    bng_acct a{};
    a.up_packets = 3, a.up_bytes = 1500, a.up_drop_packets = 7, a.up_drop_bytes = 700;
    a.down_packets = 5, a.down_bytes = 6000000000ull, a.down_drop_packets = 9, a.down_drop_bytes = 900;
    radius::SessionCounters s = radius::CountersOf(a);
    CHECK_EQ(s.InputOctets, 1500ull); // Acct-Input: from the user, upstream, passed frames only
    CHECK_EQ(s.InputPackets, 3ull);
    CHECK_EQ(s.OutputOctets, 6000000000ull);
    CHECK_EQ(s.OutputPackets, 5ull);
}

static void test_fetcher() {
    const uint32_t ip = key(10, 0, 0, 7);
    auto addr_of = [&](const std::string &id) -> std::optional<uint32_t> {
        if (id == "sess-7") return ip;
        if (id == "sess-gone") return key(10, 0, 0, 8);
        return std::nullopt;
    };
    auto reader = [&](uint32_t a, bng_acct *out) {
        if (a != ip) return -ENOENT;
        *out = bng_acct{};
        out->up_bytes = 42, out->up_packets = 1, out->down_bytes = 84, out->down_packets = 2;
        return 0;
    };
    radius::CounterFetcher f = radius::MakeCounterFetcher(addr_of, reader);
    auto r = f("sess-7");
    CHECK_EQ(r.ok(), true);
    CHECK_EQ(r->InputOctets, 42ull);
    CHECK_EQ(r->OutputPackets, 2ull);
    CHECK_EQ(f("sess-gone").ok(), false); // the address has no record
    CHECK_EQ(f("unknown").ok(), false);   // no address for the session
    // a context that is not open: the read is refused, not a zero record
    auto none = std::make_shared<Backend>();
    CHECK_EQ(radius::ContextReader(none)(ip, nullptr) < 0, true);
}

static void test_shard_routing() {
    for (uint32_t world : {2u, 8u}) {
        auto dir = std::make_shared<shard::Directory>(world);
        std::vector<std::shared_ptr<Backend>> shards;
        for (uint32_t i = 0; i < world; i++) shards.push_back(std::make_shared<Backend>()); // never opened
        shard::Router r(shards, dir);
        for (uint32_t s = 0; s < 64; s++) {
            const uint64_t mac = 0x020000000000ull + s * 0x10001ull;
            const uint32_t ip = key(10, 1, (uint8_t)(s >> 8), (uint8_t)s);
            dir->Learn(mac, ip);
            CHECK_EQ(r.AcctOwner(ip), (int)bng_shard_of_mac(mac, world));
        }
        bng_acct out{};
        CHECK_EQ(r.AcctOwner(key(192, 0, 2, 1)), -ENOENT); // never leased: no owner
        CHECK_EQ(r.AcctRead(key(192, 0, 2, 1), &out), -ENOENT);
        dir->Forget(0x020000000000ull);
        CHECK_EQ(r.AcctOwner(key(10, 1, 0, 0)), -ENOENT);
    }
}

// one qos_ingress_prog frame from 10.9.0.1, counted and read back through the counter source
static void test_gpu_roundtrip() {
    auto b = Backend::Open();
    if (!b->ctx) {
        fprintf(stderr, "FAIL bng_open: %s\n", b->open_error.c_str());
        g_fail++;
        return;
    }
    const uint32_t ip = key(10, 9, 0, 1);
    uint8_t bucket[32] = {0}; // rate 0: unlimited
    CHECK_EQ(bng_map_update(b->ctx, bng_map_id(b->ctx, "qos_ingress"), &ip, bucket, BNG_ANY), 0);
    const int prog = bng_prog_id(b->ctx, "qos_ingress_prog");
    CHECK_EQ(bng_acct_enable(b->ctx, prog, 1), 0);
    CHECK_EQ(bng_acct_enable(b->ctx, bng_prog_id(b->ctx, "antispoof_ingress"), 1), -EOPNOTSUPP);
    CHECK_EQ(bng_acct_enable(b->ctx, 99, 1), -EINVAL);
    uint8_t frame[64] = {0};
    frame[12] = 0x08, frame[14] = 0x45, frame[23] = 17;
    memcpy(frame + 26, &ip, 4);
    uint32_t len = 60;
    uint8_t verdict = 0xff;
    bng_batch bt{};
    bt.pkts = frame, bt.len = &len, bt.verdict = &verdict, bt.n = 1, bt.stride = 64, bt.mem = BNG_MEM_HOST, bt.arena_bytes = 4;
    CHECK_EQ(bng_prog_run(b->ctx, prog, &bt), 0);
    CHECK_EQ(bng_prog_run(b->ctx, prog, &bt), 0);
    auto f = radius::MakeCounterFetcher([&](const std::string &) -> std::optional<uint32_t> { return ip; }, radius::ContextReader(b));
    auto r = f("s");
    CHECK_EQ(r.ok(), true);
    if (r.ok()) {
        CHECK_EQ(r->InputOctets, 120ull);
        CHECK_EQ(r->InputPackets, 2ull);
        CHECK_EQ(r->OutputOctets, 0ull);
    }
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    test_layout();
    test_counter_mapping();
    test_fetcher();
    test_shard_routing();
    if (mode == "gpu") test_gpu_roundtrip();
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
