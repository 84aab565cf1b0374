// Tests of the host side of idle detection: idle::Monitor (bng_host.hpp) against a fake dataplane and a fake clock,
// and the fan-out of shard::Router::IdleTimeoutSet / IdleScan / IdleRead (bng_shard.hpp).
// `test_idle_host cpu` needs no device; `test_idle_host gpu` also runs the Monitor and a 2-shard Router on dataplane
// contexts, with frames stamping the records.
#include <cstddef>
#include <cstdio>
#include <map>
#include <string>
#include <vector>

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

static const uint64_t S = 1000000000ull;

static void test_layout() {
    CHECK_EQ(sizeof(bng_idle), (size_t)32);
    CHECK_EQ(offsetof(bng_idle, down_ns), (size_t)8);
    CHECK_EQ(offsetof(bng_idle, since_ns), (size_t)16);
    CHECK_EQ(offsetof(bng_idle, timeout_s), (size_t)24);
    CHECK_EQ(offsetof(bng_idle, flags), (size_t)28);
}

// The dataplane's rule, restated on the host: records of the addresses with an entry, stamped by hand.
struct FakeDataplane {
    struct Rec {
        std::optional<uint64_t> up, down, since;
        uint32_t timeout = 0;
    };
    std::map<uint32_t, Rec> recs;
    int scans = 0;
    int Set(const uint32_t *a, const uint32_t *t, uint64_t n, int32_t *res) {
        for (uint64_t i = 0; i < n; i++) {
            auto it = recs.find(a[i]);
            res[i] = it == recs.end() ? -ENOENT : 0;
            if (it != recs.end()) it->second.timeout = t[i];
        }
        return 0;
    }
    int64_t Scan(uint64_t now, uint32_t def, uint32_t flags, uint32_t *ao, bng_idle *o, uint64_t cap) {
        scans++;
        int64_t n = 0;
        for (auto &kv : recs) {
            Rec &r = kv.second;
            if (!r.since) {
                r.since = now;
                continue;
            }
            uint64_t ref = *r.since;
            if ((flags & BNG_IDLE_UP) && r.up) ref = std::max(ref, *r.up);
            if ((flags & BNG_IDLE_DOWN) && r.down) ref = std::max(ref, *r.down);
            const uint32_t t = r.timeout ? r.timeout : def;
            if (t == BNG_IDLE_NEVER || ref > now || now - ref <= (uint64_t)t * S) continue;
            if ((uint64_t)n < cap) {
                ao[n] = kv.first;
                o[n] = bng_idle{r.up.value_or(0), r.down.value_or(0), *r.since, r.timeout,
                                (r.up ? BNG_IDLE_UP : 0u) | (r.down ? BNG_IDLE_DOWN : 0u) | BNG_IDLE_STARTED};
            }
            n++;
        }
        return n;
    }
};

static void test_monitor() {
    FakeDataplane dp;
    uint64_t now = 1000 * S;
    std::vector<std::pair<std::string, std::string>> terminated;
    idle::Monitor::Config cfg;
    cfg.default_idle_timeout_s = 600;
    idle::Monitor m([&](const uint32_t *a, const uint32_t *t, uint64_t n, int32_t *r) { return dp.Set(a, t, n, r); },
                    [&](uint64_t nw, uint32_t d, uint32_t f, uint32_t *a, bng_idle *o, uint64_t c) { return dp.Scan(nw, d, f, a, o, c); },
                    [&](const std::string &s, const std::string &why) { terminated.emplace_back(s, why); }, [&] { return now; }, cfg);
    const uint32_t a1 = key(10, 0, 0, 1), a2 = key(10, 0, 0, 2), a3 = key(10, 0, 0, 3), a4 = key(10, 0, 0, 4), a5 = key(10, 0, 0, 5);
    for (uint32_t a : {a1, a2, a3, a4, a5}) dp.recs[a] = {};
    dp.recs[key(10, 0, 0, 9)] = {}; // a subscriber without a session: never armed, never reported
    CHECK_EQ((bool)m.OnAccept("s1", a1), false);      // the default: 600 s
    CHECK_EQ((bool)m.OnAccept("s2", a2, 60u), false); // Idle-Timeout 60 s from Access-Accept
    CHECK_EQ((bool)m.OnAccept("s3", a3, 0u), false);  // attribute present but 0: the default
    CHECK_EQ((bool)m.OnAccept("s4", a4, 60u), false);
    CHECK_EQ((bool)m.OnAccept("s5", a5, 60u), false);
    CHECK_EQ((bool)m.OnAccept("s6", key(10, 0, 0, 6), 60u), true); // no entry for the address: the error comes back
    CHECK_EQ(dp.recs[a1].timeout, 600u);
    CHECK_EQ(dp.recs[a2].timeout, 60u);
    CHECK_EQ(dp.recs[a3].timeout, 600u);
    CHECK_EQ((bool)m.OnCoA("s5", 0), false); // CoA: Idle-Timeout 0 disables the check
    CHECK_EQ(dp.recs[a5].timeout, BNG_IDLE_NEVER);
    CHECK_EQ((bool)m.OnCoA("nobody", 5), true);
    CHECK_EQ(m.Tick(), (int64_t)0); // the first tick starts every record
    CHECK_EQ(terminated.size(), (size_t)0);
    now += 30 * S;
    dp.recs[a4].up = now; // s4 sends
    now += 31 * S;        // 61 s after the start: s2 is idle, s4 was active 31 s ago
    CHECK_EQ(m.Tick(), (int64_t)1);
    CHECK_EQ(terminated.size(), (size_t)1);
    if (terminated.size() == 1) {
        CHECK_EQ(terminated[0].first == "s2", true);
        CHECK_EQ(terminated[0].second == "idle_timeout", true);
    }
    CHECK_EQ(m.Tick(), (int64_t)0); // once: s2 is not terminated again, though its entries are still there
    CHECK_EQ(dp.recs[a2].timeout, BNG_IDLE_NEVER);
    now += 30 * S; // s4: 61 s since its last frame; exactly 60 s would not be idle (">", as the reference)
    dp.recs[a4].down = now - 60 * S;
    CHECK_EQ(m.Tick(), (int64_t)0);
    now += 1;
    CHECK_EQ(m.Tick(), (int64_t)1);
    CHECK_EQ(terminated.back().first == "s4", true);
    now += 600 * S; // s1 and s3 reach the default; s5 never; the subscriber without a session is never reported
    CHECK_EQ(m.Tick(), (int64_t)2);
    CHECK_EQ(terminated.size(), (size_t)4);
    CHECK_EQ(m.Sessions(), (size_t)1);
    m.Forget("s5");
    CHECK_EQ(m.Sessions(), (size_t)0);
    // a full output: the Monitor asks again with room for everything the scan found
    FakeDataplane big;
    std::vector<std::pair<std::string, std::string>> t2;
    uint64_t clk = 0;
    idle::Monitor m2([&](const uint32_t *a, const uint32_t *t, uint64_t n, int32_t *r) { return big.Set(a, t, n, r); },
                     [&](uint64_t nw, uint32_t d, uint32_t f, uint32_t *a, bng_idle *o, uint64_t c) { return big.Scan(nw, d, f, a, o, c); },
                     [&](const std::string &s, const std::string &) { t2.emplace_back(s, ""); }, [&] { return clk; }, cfg);
    for (uint32_t i = 0; i < 200; i++) {
        big.recs[key(10, 1, 0, (uint8_t)i)] = {};
        m2.OnAccept("b" + std::to_string(i), key(10, 1, 0, (uint8_t)i), 1u);
    }
    m2.Tick();
    clk += 2 * S;
    CHECK_EQ(m2.Tick(), (int64_t)200);
    CHECK_EQ(t2.size(), (size_t)200);
}

static void test_router_cpu() {
    for (uint32_t world : {2u, 8u}) {
        auto dir = std::make_shared<shard::Directory>(world);
        std::vector<std::shared_ptr<Backend>> shards;
        for (uint32_t i = 0; i < world; i++) shards.push_back(std::make_shared<Backend>()); // never opened
        shard::Router r(shards, dir);
        const uint32_t a = key(10, 2, 0, 1);
        dir->Learn(0x020000000001ull, a);
        uint32_t t = 5;
        int32_t res = 0;
        bng_idle rec{};
        uint32_t ao = 0;
        // every call reaches a context and reports its refusal
        CHECK_EQ(r.IdleTimeoutSet(&a, &t, 1, &res), -EINVAL);
        CHECK_EQ(r.IdleRead(&a, 1, &rec, &res), -EINVAL);
        CHECK_EQ(r.IdleScan(0, 0, BNG_IDLE_UP, &ao, &rec, 1), (int64_t)-EINVAL);
        CHECK_EQ(r.IdleScan(0, 0, BNG_IDLE_UP, nullptr, nullptr, 1), (int64_t)-EINVAL);
        CHECK_EQ(r.IdleTimeoutSet(nullptr, nullptr, 0, nullptr), 0);
    }
}

// ---- on a device ----
static int run_frame(bng_ctx *c, int prog, uint32_t src, uint64_t now) {
    uint8_t frame[64] = {0};
    frame[12] = 0x08, frame[14] = 0x45, frame[23] = 17;
    memcpy(frame + 26, &src, 4);
    uint32_t len = 60;
    uint8_t verdict = 0xff;
    bng_batch bt{};
    bt.pkts = frame, bt.len = &len, bt.verdict = &verdict, bt.n = 1, bt.stride = 64, bt.mem = BNG_MEM_HOST, bt.arena_bytes = 4, bt.now_ns = now;
    return bng_prog_run(c, prog, &bt);
}

static void test_gpu() {
    bng_open_opts o{};
    o.struct_size = sizeof(o), o.device = -1, o.max_batch = 1024, o.max_subscribers = 1024, o.max_nat_sessions = 4096,
    o.max_eim_mappings = 4096;
    std::vector<std::shared_ptr<Backend>> shards = {Backend::Open(&o), Backend::Open(&o)};
    for (auto &b : shards)
        if (!b->ctx) {
            fprintf(stderr, "FAIL bng_open: %s\n", b->open_error.c_str());
            g_fail++;
            return;
        }
    auto dir = std::make_shared<shard::Directory>(2);
    shard::Router r(shards, dir);
    // 16 subscribers, each on the shard its MAC gives; qos_ingress entries only on the owner
    std::vector<uint32_t> addrs;
    std::vector<int> owner;
    for (uint32_t s = 0; s < 16; s++) {
        const uint64_t mac = 0x020000000100ull + s;
        const uint32_t a = key(10, 3, 0, (uint8_t)(s + 1));
        dir->Learn(mac, a);
        addrs.push_back(a);
        owner.push_back((int)bng_shard_of_mac(mac, 2));
        uint8_t bucket[32] = {0};
        bng_ctx *c = shards[(size_t)owner.back()]->ctx;
        CHECK_EQ(bng_map_update(c, bng_map_id(c, "qos_ingress"), &a, bucket, BNG_ANY), 0);
    }
    const int prog = bng_prog_id(shards[0]->ctx, "qos_ingress_prog");
    for (auto &b : shards) CHECK_EQ(bng_idle_enable(b->ctx, prog, 1), 0);
    std::vector<uint32_t> t(16, 10);
    std::vector<int32_t> res(16, 1);
    CHECK_EQ(r.IdleTimeoutSet(addrs.data(), t.data(), 16, res.data()), 0);
    for (int32_t x : res) CHECK_EQ(x, 0);
    const uint32_t stranger = key(192, 0, 2, 1); // no owner known, no entry anywhere
    uint32_t t1 = 3;
    int32_t r1 = 0;
    CHECK_EQ(r.IdleTimeoutSet(&stranger, &t1, 1, &r1), 0);
    CHECK_EQ(r1, -ENOENT);
    // the Monitor over the router: sessions of the even subscribers only
    uint64_t now = 5 * S;
    std::vector<std::string> gone;
    idle::Monitor m(r.IdleTimeoutSetter(), r.IdleScanner(), [&](const std::string &s, const std::string &why) {
        CHECK_EQ(why == idle::kReasonIdleTimeout, true);
        gone.push_back(s);
    }, [&] { return now; });
    for (uint32_t s = 0; s < 16; s += 2) CHECK_EQ((bool)m.OnAccept("s" + std::to_string(s), addrs[s], 10u), false);
    CHECK_EQ(m.Tick(), (int64_t)0); // starts every record at 5 s
    now = 12 * S;
    for (uint32_t s = 0; s < 8; s++) CHECK_EQ(run_frame(shards[(size_t)owner[s]]->ctx, prog, addrs[s], now), 0); // 0..7 active at 12 s
    std::vector<bng_idle> recs(16);
    CHECK_EQ(r.IdleRead(addrs.data(), 16, recs.data(), res.data()), 0);
    for (uint32_t s = 0; s < 16; s++) {
        CHECK_EQ(res[s], 0);
        CHECK_EQ(recs[s].since_ns, 5 * S);
        CHECK_EQ(recs[s].up_ns, s < 8 ? now : 0);
        CHECK_EQ(recs[s].flags, (s < 8 ? BNG_IDLE_UP : 0u) | BNG_IDLE_STARTED);
    }
    now = 16 * S; // 11 s after the start: 8..15 are idle; only the even ones have sessions
    CHECK_EQ(m.Tick(), (int64_t)4);
    CHECK_EQ(gone.size(), (size_t)4);
    CHECK_EQ(m.Tick(), (int64_t)0);
    std::vector<uint32_t> ao(16);
    CHECK_EQ(r.IdleScan(now, 0, BNG_IDLE_UP | BNG_IDLE_DOWN, ao.data(), recs.data(), 16), (int64_t)4); // the odd 9..15
    CHECK_EQ(r.IdleScan(now, 0, BNG_IDLE_UP, ao.data(), recs.data(), 1), (int64_t)4);                 // found, 1 written
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    test_layout();
    test_monitor();
    test_router_cpu();
    if (mode == "gpu") test_gpu();
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
