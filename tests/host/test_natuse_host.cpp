// Tests of the host side of the NAT port-usage census: nat::UsageMonitor (bng_host.hpp) against a fake census, and
// shard::Router::MergeNatUsage (bng_shard.hpp).  `test_natuse_host cpu` needs no device; `test_natuse_host gpu` also
// runs nat::Manager::PortUsage and a 2-shard Router::NatUsage on dataplane contexts filled through bng_map_update.
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

static void test_layout() {
    CHECK_EQ(sizeof(bng_nat_sub_use), (size_t)64);
    CHECK_EQ(offsetof(bng_nat_sub_use, public_ip), (size_t)16);
    CHECK_EQ(offsetof(bng_nat_sub_use, in_use), (size_t)24);
    CHECK_EQ(offsetof(bng_nat_sub_use, permille), (size_t)48);
    CHECK_EQ(sizeof(bng_nat_pub_use), (size_t)64);
    CHECK_EQ(offsetof(bng_nat_pub_use, blocks), (size_t)24);
    CHECK_EQ(offsetof(bng_nat_pub_use, unreachable), (size_t)44);
    CHECK_EQ(sizeof(bng_nat_usage_sum), (size_t)80);
}

// A census the test sets by hand: the subscribers' and public addresses' permille, filtered as bng_nat_usage filters.
struct FakeCensus {
    std::map<uint32_t, uint32_t> sub_pm;                      // address -> permille
    std::map<uint32_t, std::pair<uint32_t, uint32_t>> pub_use; // address -> (max in_use, block_ports)
    uint64_t sessions = 0;
    std::vector<uint32_t> asked;
    int Run(uint32_t min_permille, nat::PortUsageReport *out) {
        asked.push_back(min_permille);
        *out = nat::PortUsageReport{};
        for (auto &kv : sub_pm) {
            if (kv.second < min_permille) continue;
            bng_nat_sub_use r{};
            r.permille = kv.second;
            r.block_ports = 1000;
            r.in_use[1] = kv.second;
            r.in_use_any = kv.second + 1;
            out->SubAddrs.push_back(kv.first);
            out->Subs.push_back(r);
        }
        for (auto &kv : pub_use) {
            bng_nat_pub_use r{};
            r.in_use[2] = kv.second.first;
            r.in_use_any = kv.second.first + 7;
            r.block_ports = kv.second.second;
            out->PubAddrs.push_back(kv.first);
            out->Pubs.push_back(r);
        }
        out->Summary.sessions = sessions;
        out->Summary.subs_found = out->Subs.size();
        out->Summary.pubs_found = out->Pubs.size();
        return 0;
    }
};

static void test_monitor_crossings() {
    FakeCensus f;
    std::map<uint32_t, uint32_t> ports_used;
    uint64_t bindings = 0;
    std::vector<nat::UsageAlert> alerts;
    nat::UsageMonitor m([&](uint32_t mp, nat::PortUsageReport *o) { return f.Run(mp, o); },
                        [&](uint32_t a, uint32_t n) { ports_used[a] = n; }, [&](uint64_t n) { bindings = n; },
                        [&](const nat::UsageAlert &a) { alerts.push_back(a); });
    const uint32_t A = key(10, 0, 0, 1), B = key(10, 0, 0, 2), P = key(203, 0, 113, 1);
    auto tick = [&]() {
        alerts.clear();
        CHECK_EQ((bool)m.Tick().err, false);
    };
    f.sub_pm = {{A, 100}, {B, 799}};
    f.pub_use = {{P, {100, 1000}}};
    f.sessions = 42;
    tick();
    CHECK_EQ(alerts.size(), (size_t)0);
    CHECK_EQ(f.asked.back(), 800u); // only subscribers at or above the warning level are copied out
    CHECK_EQ(ports_used[P], 107u);
    CHECK_EQ(bindings, (uint64_t)42);
    f.sub_pm[B] = 800; // crosses the warning level: one alert
    tick();
    CHECK_EQ(alerts.size(), (size_t)1);
    CHECK_EQ(alerts[0].Addr, B);
    CHECK_EQ((int)alerts[0].Level, (int)nat::UsageLevel::Warning);
    CHECK_EQ(alerts[0].Public, false);
    tick(); // stays above: no new alert
    CHECK_EQ(alerts.size(), (size_t)0);
    f.sub_pm[B] = 950; // warning -> critical: one alert
    f.sub_pm[A] = 1000; // ok -> critical at once: one alert, at the critical level
    tick();
    CHECK_EQ(alerts.size(), (size_t)2);
    for (auto &a : alerts) CHECK_EQ((int)a.Level, (int)nat::UsageLevel::Critical);
    CHECK_EQ((int)m.SubscriberLevel(A), (int)nat::UsageLevel::Critical);
    f.sub_pm[B] = 850; // falls back to warning: silent, and re-arms the critical level
    tick();
    CHECK_EQ(alerts.size(), (size_t)0);
    CHECK_EQ((int)m.SubscriberLevel(B), (int)nat::UsageLevel::Warning);
    f.sub_pm[B] = 900;
    tick();
    CHECK_EQ(alerts.size(), (size_t)1);
    f.sub_pm[A] = 10; // leaves the report: back to ok, and a later rise alerts again
    tick();
    CHECK_EQ((int)m.SubscriberLevel(A), (int)nat::UsageLevel::Ok);
    f.sub_pm[A] = 820;
    tick();
    CHECK_EQ(alerts.size(), (size_t)1);
    CHECK_EQ(alerts[0].Addr, A);
    // public addresses: the same rule on max(in_use) / block_ports; no ports: never alerts
    f.pub_use[P] = {910, 1000};
    f.pub_use[key(0, 0, 0, 0)] = {5, 0};
    tick();
    CHECK_EQ(alerts.size(), (size_t)1);
    CHECK_EQ(alerts[0].Public, true);
    CHECK_EQ(alerts[0].Permille, 910u);
    CHECK_EQ((int)m.PublicLevel(P), (int)nat::UsageLevel::Critical);
    // a failing census is an error, and changes no level
    nat::UsageMonitor bad([](uint32_t, nat::PortUsageReport *) { return -EIO; }, [](uint32_t, uint32_t) {}, [](uint64_t) {},
                          [](const nat::UsageAlert &) {});
    CHECK_EQ((bool)bad.Tick().err, true);
}

static void test_merge() {
    std::vector<nat::PortUsageReport> parts(2);
    const uint32_t P = key(203, 0, 113, 1), Q = key(203, 0, 113, 2);
    for (int k = 0; k < 2; k++) {
        auto &p = parts[k];
        p.Summary.subscribers = 3 + k, p.Summary.sessions = 10 * (k + 1), p.Summary.triples = 5, p.Summary.unreachable = k;
        p.Summary.subs_found = 1, p.Summary.pubs_found = 1 + k;
        bng_nat_sub_use s{};
        s.sessions = 7 + k;
        p.SubAddrs.push_back(key(10, 0, 0, (uint8_t)(1 + k)));
        p.Subs.push_back(s);
        bng_nat_pub_use u{};
        u.sessions = 4 + k, u.eim = 1, u.block_ports = 1024, u.blocks = 1, u.in_use[0] = 3, u.in_use_any = 3 + k, u.unreachable = k;
        p.PubAddrs.push_back(P);
        p.Pubs.push_back(u);
        if (k == 1) {
            p.PubAddrs.push_back(Q);
            p.Pubs.push_back(u);
        }
    }
    nat::PortUsageReport m = shard::Router::MergeNatUsage(parts);
    CHECK_EQ(m.Summary.subscribers, (uint64_t)7);
    CHECK_EQ(m.Summary.sessions, (uint64_t)30);
    CHECK_EQ(m.Summary.triples, (uint64_t)10); // a triple held on two shards counts once per shard
    CHECK_EQ(m.Summary.unreachable, (uint64_t)1);
    CHECK_EQ(m.Summary.subs_found, (uint64_t)2);
    CHECK_EQ(m.Summary.pubs_found, (uint64_t)2);
    CHECK_EQ(m.SubAddrs.size(), (size_t)2);
    CHECK_EQ(m.PubAddrs.size(), (size_t)2);
    for (size_t i = 0; i < m.PubAddrs.size(); i++) {
        const bng_nat_pub_use &u = m.Pubs[i];
        if (m.PubAddrs[i] == P) {
            CHECK_EQ(u.sessions, (uint64_t)9);
            CHECK_EQ(u.eim, (uint64_t)2);
            CHECK_EQ(u.block_ports, (uint64_t)2048);
            CHECK_EQ(u.blocks, 2u);
            CHECK_EQ(u.in_use[0], 6u);
            CHECK_EQ(u.in_use_any, 7u);
            CHECK_EQ(u.unreachable, 1u);
        } else {
            CHECK_EQ(m.PubAddrs[i], Q);
            CHECK_EQ(u.sessions, (uint64_t)5);
        }
    }
}

// ---- on the GPU ----
static void put_sub(bng_ctx *c, uint32_t addr, uint32_t pub, uint16_t ps, uint16_t pe) {
    nat::SubscriberNAT v{};
    v.Block.PublicIP = pub, v.Block.PortStart = ps, v.Block.PortEnd = pe, v.Block.NextPort = ps;
    CHECK_EQ(bng_map_update(c, bng_map_id(c, "subscriber_nat"), &addr, &v, BNG_ANY), 0);
}
static void put_session(bng_ctx *c, uint32_t src, uint16_t sport_be, uint32_t nat_ip, uint16_t nat_port_be, uint8_t proto) {
    nat::NATKey k{};
    k.SrcIP = src, k.DstIP = key(8, 8, 8, 8), k.SrcPort = sport_be, k.DstPort = 0x5000, k.Protocol = proto;
    nat::NATSession s{};
    s.NATIP = nat_ip, s.NATPort = nat_port_be, s.Protocol = proto;
    CHECK_EQ(bng_map_update(c, bng_map_id(c, "nat_sessions"), &k, &s, BNG_ANY), 0);
}

static void test_gpu() {
    bng_open_opts o{};
    o.struct_size = sizeof(o), o.device = -1, o.max_subscribers = 1024, o.max_nat_sessions = 4096, o.max_eim_mappings = 4096;
    o.max_batch = 1024;
    std::vector<std::shared_ptr<Backend>> shards;
    for (int k = 0; k < 2; k++) {
        shards.push_back(Backend::Open(&o));
        if (!shards.back()->ctx) {
            fprintf(stderr, "FAIL bng_open: %s\n", shards.back()->open_error.c_str());
            g_fail++;
            return;
        }
    }
    const uint32_t P = key(203, 0, 113, 1);
    // shard 0: subscriber A with 4 ports, 2 TCP sessions; shard 1: subscriber B on the same address
    put_sub(shards[0]->ctx, key(10, 0, 0, 1), P, 1000, 1003);
    put_session(shards[0]->ctx, key(10, 0, 0, 1), 0x0100, P, 0xE803, 6); // nat port 1000
    put_session(shards[0]->ctx, key(10, 0, 0, 1), 0x0200, P, 0xE903, 6); // 1001
    put_sub(shards[1]->ctx, key(10, 0, 0, 2), P, 2000, 2009);
    put_session(shards[1]->ctx, key(10, 0, 0, 2), 0x0100, P, 0xD007, 17); // 2000
    nat::PortUsageReport one;
    CHECK_EQ(nat::ContextPortUsage(shards[0]->ctx, 0, &one), 0);
    CHECK_EQ(one.Subs.size(), (size_t)1);
    if (!one.Subs.empty()) {
        CHECK_EQ(one.Subs[0].in_use[0], 2u);
        CHECK_EQ(one.Subs[0].permille, 500u);
        CHECK_EQ(one.Subs[0].unreachable, 2u); // no reverse entries
    }
    auto dir = std::make_shared<shard::Directory>(2);
    shard::Router r(shards, dir);
    nat::PortUsageReport all;
    CHECK_EQ(r.NatUsage(0, &all), 0);
    CHECK_EQ(all.Summary.subscribers, (uint64_t)2);
    CHECK_EQ(all.Summary.sessions, (uint64_t)3);
    CHECK_EQ(all.PubAddrs.size(), (size_t)1);
    if (!all.Pubs.empty()) {
        CHECK_EQ(all.Pubs[0].blocks, 2u);
        CHECK_EQ(all.Pubs[0].block_ports, (uint64_t)14);
        CHECK_EQ(all.Pubs[0].in_use_any, 3u);
    }
    // the manager's census keeps GetAllocation's PortsInUse
    nat::ManagerConfig mc;
    mc.Interface = "eth0";
    mc.Backend_ = shards[0];
    mc.PortsPerSubscriber = 4;
    mc.PortRangeStart = 1000;
    auto mgr = *nat::Manager::NewManager(mc).value;
    CHECK_EQ((bool)mgr->Start(), false);
    CHECK_EQ((bool)mgr->AddPublicIP(IP{203, 0, 113, 1}), false);
    auto a = mgr->AllocateNAT(IP{10, 0, 0, 1});
    CHECK_EQ((bool)a.err, false);
    CHECK_EQ(mgr->GetAllocation(IP{10, 0, 0, 1})->PortsInUse, 0u);
    // the manager keys its maps by Backend::AddrKey of the address as a big-endian number
    const uint32_t priv = shards[0]->AddrKey(0x0A000001u), pub = shards[0]->AddrKey(0xCB007101u);
    put_session(shards[0]->ctx, priv, 0x0300, pub, 0xE803, 17); // 1000
    put_session(shards[0]->ctx, priv, 0x0400, pub, 0xEA03, 6);  // 1002
    auto rep = mgr->PortUsage();
    CHECK_EQ((bool)rep.err, false);
    CHECK_EQ(mgr->GetAllocation(IP{10, 0, 0, 1})->PortsInUse, 2u);
}

int main(int argc, char **argv) {
    const std::string mode = argc > 1 ? argv[1] : "cpu";
    test_layout();
    test_monitor_crossings();
    test_merge();
    if (mode == "gpu") test_gpu();
    printf("%d checks, %d failures\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
