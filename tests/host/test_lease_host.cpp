// DHCP lease census and sweep, host side: dhcp::PoolMonitor's threshold crossings, dhcp::Server::CleanupExpiredLeases'
// loop against a fake sweep, shard::Router's merge (cpu); Loader / Router against one and two contexts (gpu).
#include <cstdio>
#include <cstring>
#include <memory>

#include "../../bng_b200/host/bng_dhcp_slow.hpp"
#include "../../bng_b200/host/bng_shard.hpp"

using namespace bng;

static int failures = 0;
#define CHECK(c)                                                            \
    do {                                                                    \
        if (!(c)) {                                                         \
            printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c);             \
            failures++;                                                     \
        }                                                                   \
    } while (0)

static void test_sizes() {
    CHECK(sizeof(bng_lease_pool_use) == 64);
    CHECK(sizeof(bng_lease_removed) == 64);
    CHECK(sizeof(bng_lease_sum) == 88);
    CHECK(offsetof(bng_lease_removed, lease_expiry) == 32 && offsetof(bng_lease_removed, map) == 52);
    CHECK(offsetof(bng_lease_pool_use, addrs) == 32 && offsetof(bng_lease_pool_use, known) == 52);
}

static void test_pool_monitor() {
    uint32_t permille = 0, conflicts = 0;
    auto census = [&](uint64_t, ebpf::LeaseCensusReport *out) {
        out->PoolIDs = {1, 9};
        out->Pools.assign(2, bng_lease_pool_use{});
        out->Pools[0].known = 1, out->Pools[0].permille = permille, out->Pools[0].conflicts = conflicts;
        out->Pools[1].permille = 1000; // unknown pool: no gauge, no level
        out->Summary.entries[0] = 42;
        return 0;
    };
    std::vector<dhcp::PoolAlert> alerts;
    std::map<uint32_t, uint32_t> gauge;
    uint64_t active = 0;
    dhcp::PoolMonitor mon(census, [&](uint32_t p, uint32_t v) { gauge[p] = v; }, [&](uint64_t n) { active = n; },
                          [&](const dhcp::PoolAlert &a) { alerts.push_back(a); });
    permille = 799;
    CHECK(mon.Tick(0).ok() && alerts.empty() && gauge.size() == 1 && gauge[1] == 799 && active == 42);
    permille = 800;
    CHECK(mon.Tick(0).ok() && alerts.size() == 1 && alerts[0].Level == dhcp::PoolLevel::Warning);
    CHECK(mon.Tick(0).ok() && alerts.size() == 1); // stays above: no second alert
    permille = 900;
    CHECK(mon.Tick(0).ok() && alerts.size() == 2 && alerts[1].Level == dhcp::PoolLevel::Critical);
    permille = 850;
    CHECK(mon.Tick(0).ok() && alerts.size() == 2 && mon.Level(1) == dhcp::PoolLevel::Warning);
    permille = 100;
    CHECK(mon.Tick(0).ok() && mon.Level(1) == dhcp::PoolLevel::Ok);
    permille = 950;
    CHECK(mon.Tick(0).ok() && alerts.size() == 3 && alerts[2].Level == dhcp::PoolLevel::Critical);
    permille = 0, conflicts = 2;
    CHECK(mon.Tick(0).ok() && alerts.size() == 4 && alerts[3].Level == dhcp::PoolLevel::Ok && alerts[3].Conflicts == 2);
}

static void test_cleanup_loop() {
    dhcp::PoolManager pm;
    dhcp::PoolConfig pc;
    pc.ID = 1, pc.Name = "p", pc.Network = "10.0.0.0/24", pc.Gateway = "10.0.0.1", pc.LeaseTimeSec = 60;
    auto pool = dhcp::Pool::New(pc);
    CHECK(pool.ok());
    pm.AddPool(*pool.value);
    dhcp::Server srv(0x0A0000FE, &pm, nullptr, [] { return (int64_t)1000; });
    std::vector<bng_lease_removed> due;
    for (uint32_t i = 0; i < 5; i++) {
        const uint64_t mac = 0x020000000000ull + i;
        auto ip = (*pool.value)->Allocate(mac);
        CHECK(ip.ok());
        dhcp::Lease l;
        l.MAC = mac, l.IP = *ip.value, l.PoolID = 1, l.ExpiresAt = i == 4 ? 5000 : 100; // the last one was renewed
        srv.InstallLease(l);
        bng_lease_removed r{};
        memcpy(r.key, &mac, 8);
        r.lease_expiry = 100, r.pool_id = 1, r.allocated_ip = *ip.value, r.map = 0;
        due.push_back(r);
        if (i == 0) { // its VLAN entry went too: must not release the address a second time or drop anything else
            r.map = 1;
            due.push_back(r);
        }
    }
    const int before = (*pool.value)->Stats().Allocated;
    size_t at = 0;
    int calls = 0;
    auto sweep = [&](uint64_t, uint32_t, uint64_t cap, std::vector<bng_lease_removed> *out) -> int64_t {
        calls++;
        const int64_t found = (int64_t)(due.size() - at);
        out->clear();
        while (at < due.size() && out->size() < cap) out->push_back(due[at++]);
        return found;
    };
    CHECK(srv.CleanupExpiredLeases(2000ull * 1000000000ull, sweep, 2) == 6);
    CHECK(calls == 3 && srv.ActiveLeases() == 1);
    CHECK((*pool.value)->Stats().Allocated == before - 4);
    // a removed entry without a lease whose address another client holds by now: that allocation stays
    auto other = (*pool.value)->Allocate(0x02CC00000001ull);
    CHECK(other.ok());
    bng_lease_removed stale{};
    const uint64_t gone_mac = 0x02DD00000001ull;
    memcpy(stale.key, &gone_mac, 8);
    stale.lease_expiry = 100, stale.pool_id = 1, stale.allocated_ip = *other.value, stale.map = 0;
    due.assign(1, stale), at = 0;
    const int held = (*pool.value)->Stats().Allocated;
    CHECK(srv.CleanupExpiredLeases(2000ull * 1000000000ull, sweep, 2) == 1);
    CHECK((*pool.value)->Stats().Allocated == held);
    auto bad = [](uint64_t, uint32_t, uint64_t, std::vector<bng_lease_removed> *) -> int64_t { return -EIO; };
    CHECK(srv.CleanupExpiredLeases(0, bad) == -EIO);
}

static void test_merge() {
    std::vector<ebpf::LeaseCensusReport> parts(2);
    for (int k = 0; k < 2; k++) {
        parts[k].PoolIDs = {1, (uint32_t)(7 + k)};
        parts[k].Pools.assign(2, bng_lease_pool_use{});
        parts[k].Pools[0].entries[0] = 10 + k, parts[k].Pools[0].addrs = 10 + k, parts[k].Pools[0].known = 1;
        parts[k].Pools[0].prefix_hosts = 256;
        parts[k].Summary.entries[0] = 10 + k, parts[k].Summary.addrs = 10 + k, parts[k].Summary.pools_found = 2;
    }
    auto m = shard::Router::MergeLeaseCensus(parts);
    CHECK(m.Summary.pools_found == 3 && m.PoolIDs.size() == 3 && m.PoolIDs[0] == 1);
    CHECK(m.Pools[0].entries[0] == 21 && m.Pools[0].addrs == 21 && m.Pools[0].permille == 21 * 1000 / 256);
    CHECK(m.Summary.entries[0] == 21 && m.Summary.addrs == 21);
}

static ebpf::PoolAssignment lease(uint32_t pool, uint32_t ip_wire, uint64_t expiry) {
    ebpf::PoolAssignment a;
    a.PoolID = pool, a.AllocatedIP = ip_wire, a.LeaseExpiry = expiry;
    return a;
}

// The same leases in one context and spread over two by bng_shard_of_mac: census and sweep agree.
static void test_gpu_two_shards_leases() {
    bng_open_opts o{};
    o.struct_size = sizeof(o), o.device = -1;
    o.max_subscribers = 1024, o.max_nat_sessions = 1024, o.max_eim_mappings = 1024, o.max_batch = 1024;
    auto whole = Backend::Open(&o);
    std::vector<std::shared_ptr<Backend>> shards{Backend::Open(&o), Backend::Open(&o)};
    CHECK(whole->ctx && shards[0]->ctx && shards[1]->ctx);
    if (!whole->ctx || !shards[0]->ctx || !shards[1]->ctx) return;
    auto router = std::make_unique<shard::Router>(shards, std::make_shared<shard::Directory>(2));
    for (bng_ctx *c : {whole->ctx, shards[0]->ctx, shards[1]->ctx}) // this test writes the words in wire order
        CHECK(bng_dhcp_lease_addr_order(c, BNG_LEASE_ADDR_WIRE) == 0);
    CHECK(bng_dhcp_lease_addr_order(whole->ctx, 2) == -EINVAL && bng_dhcp_lease_addr_order(nullptr, 0) == -EINVAL);
    const int n = 200;
    ebpf::IPPool p;
    p.Network = 0x0000000A, p.PrefixLen = 16; // 10.0.0.0/16, wire order
    uint32_t pid = 1;
    int pm = bng_map_id(whole->ctx, "ip_pools"), sm = bng_map_id(whole->ctx, "subscriber_pools");
    CHECK(bng_map_update(whole->ctx, pm, &pid, &p, BNG_ANY) == 0);
    for (int k = 0; k < 2; k++) CHECK(bng_map_update(shards[k]->ctx, pm, &pid, &p, BNG_ANY) == 0);
    for (int i = 0; i < n; i++) {
        uint64_t mac = 0x020000000000ull + i;
        auto a = lease(i % 3 ? 1 : 2, 0x0000000A | (uint32_t)(i + 1) << 24, i % 4 ? 1000 : 10);
        CHECK(bng_map_update(whole->ctx, sm, &mac, &a, BNG_ANY) == 0);
        CHECK(bng_map_update(shards[bng_shard_of_mac(mac, 2)]->ctx, sm, &mac, &a, BNG_ANY) == 0);
    }
    ebpf::LeaseCensusReport one, two;
    CHECK(ebpf::ContextLeaseCensus(whole->ctx, 500ull * 1000000000ull, &one) == 0);
    CHECK(router->LeaseCensus(500ull * 1000000000ull, &two) == 0);
    CHECK(memcmp(&one.Summary, &two.Summary, sizeof(one.Summary)) == 0);
    CHECK(one.PoolIDs.size() == 2 && two.PoolIDs.size() == 2);
    std::map<uint32_t, bng_lease_pool_use> a, b;
    for (size_t i = 0; i < one.PoolIDs.size(); i++) a[one.PoolIDs[i]] = one.Pools[i];
    for (size_t i = 0; i < two.PoolIDs.size(); i++) b[two.PoolIDs[i]] = two.Pools[i];
    for (auto &kv : a) CHECK(memcmp(&kv.second, &b[kv.first], sizeof(bng_lease_pool_use)) == 0);
    CHECK(one.Summary.expired[0] == 50 && a[1].known && !a[2].known && a[1].addrs_outside == 0);
    std::vector<bng_lease_removed> r1, r2;
    CHECK(ebpf::ContextLeaseSweep(whole->ctx, 500ull * 1000000000ull, 0, 1024, &r1) == 50);
    CHECK(router->LeaseSweep(500ull * 1000000000ull, 0, 1024, &r2) == 50);
    auto key = [](const bng_lease_removed &x) { uint64_t m; memcpy(&m, x.key, 8); return m; };
    std::map<uint64_t, bng_lease_removed> s1, s2;
    for (auto &x : r1) s1[key(x)] = x;
    for (auto &x : r2) s2[key(x)] = x;
    CHECK(s1.size() == 50 && s2.size() == 50);
    for (auto &kv : s1) CHECK(s2.count(kv.first) && memcmp(&kv.second, &s2[kv.first], 64) == 0);
    CHECK(router->LeaseSweep(500ull * 1000000000ull, 0, 1024, &r2) == 0 && r2.empty());
}

// The control plane's own path: PoolManager::AddPool and Server::HandleRequest fill ip_pools and subscriber_pools through
// the Loader (addresses as numeric values, the default order); the census must place every lease inside its pool, the
// monitor must see the utilisation, and the sweep's records must give the right addresses back to the pool.
static void test_gpu_server_census_and_cleanup() {
    bng_open_opts o{};
    o.struct_size = sizeof(o), o.device = -1;
    o.max_subscribers = 1024, o.max_nat_sessions = 1024, o.max_eim_mappings = 1024, o.max_batch = 1024;
    auto be = Backend::Open(&o);
    CHECK(be->ctx != nullptr);
    if (!be->ctx) return;
    auto lr = ebpf::Loader::NewLoader("eth0", be);
    CHECK(lr.ok());
    auto loader = *lr.value;
    CHECK(!loader->Load());
    dhcp::PoolManager pm(loader.get());
    dhcp::PoolConfig pc;
    pc.ID = 3, pc.Name = "p", pc.Network = "10.20.30.0/28", pc.Gateway = "10.20.30.1", pc.LeaseTimeSec = 60;
    auto pool = dhcp::Pool::New(pc);
    CHECK(pool.ok());
    pm.AddPool(*pool.value);
    CHECK(!pm.LastSyncError());
    int64_t clock = 1000;
    dhcp::Server srv(0x0A141EFE, &pm, loader.get(), [&] { return clock; });
    const uint32_t n = 13; // .2 - .14: every address of the /28 but network, gateway and broadcast
    std::map<uint64_t, uint32_t> leased;
    for (uint32_t i = 0; i < n; i++) {
        if (i == 12) clock = 1030; // the last lease outlives the first sweep
        auto d = dhcp::ClientMessage(dhcp::Discover, i, 100 + i);
        auto dm = dhcp::Message::Parse(d.data(), d.size());
        CHECK(dm.ok());
        auto off = srv.HandleDiscover(*dm);
        CHECK(off.ok());
        if (!off.ok()) return;
        auto q = dhcp::ClientMessage(dhcp::Request, i, 100 + i, off->yiaddr);
        auto qm = dhcp::Message::Parse(q.data(), q.size());
        auto ack = srv.HandleRequest(*qm);
        CHECK(ack.ok() && ack->yiaddr == off->yiaddr && !srv.LastFastPathError());
        leased[0x020000000000ull + i] = off->yiaddr;
    }
    CHECK(srv.ActiveLeases() == n && (*pool.value)->Stats().Allocated == (int)n);

    std::vector<dhcp::PoolAlert> alerts;
    std::map<uint32_t, uint32_t> gauge;
    uint64_t active = 0;
    dhcp::PoolMonitor mon([&](uint64_t now_ns, ebpf::LeaseCensusReport *out) { return ebpf::ContextLeaseCensus(be->ctx, now_ns, out); },
                          [&](uint32_t p, uint32_t v) { gauge[p] = v; }, [&](uint64_t v) { active = v; },
                          [&](const dhcp::PoolAlert &a) { alerts.push_back(a); });
    auto t = mon.Tick(1040ull * 1000000000ull);
    CHECK(t.ok());
    if (!t.ok()) return;
    CHECK(t->PoolIDs.size() == 1 && t->PoolIDs[0] == 3);
    if (t->Pools.size() == 1) {
        const bng_lease_pool_use &u = t->Pools[0];
        CHECK(u.known == 1 && u.entries[0] == n && u.addrs == n && u.addrs_outside == 0 && u.conflicts == 0);
        CHECK(u.prefix_hosts == 16 && u.permille == n * 1000 / 16);
    }
    CHECK(active == n && gauge[3] == n * 1000 / 16 && alerts.size() == 1 && alerts[0].Level == dhcp::PoolLevel::Warning);
    auto lc = loader->LeaseCensus(1040ull * 1000000000ull);
    CHECK(lc.ok() && lc->Summary.entries[0] == n && lc->Summary.unknown_pool == 0);

    // at 1075 the twelve leases of clock 1000 (expiry 1060) are due, the one of 1030 (expiry 1090) is not
    clock = 1075;
    CHECK(srv.CleanupExpiredLeases(1075ull * 1000000000ull, loader->SweepSource(), 5) == 12);
    CHECK(srv.ActiveLeases() == 1 && (*pool.value)->Stats().Allocated == 1 && (*pool.value)->Stats().Available == 12);
    auto kept = loader->GetSubscriber(0x020000000000ull + 12);
    CHECK(kept.ok() && kept->AllocatedIP == leased[0x020000000000ull + 12]);
    CHECK(!loader->GetSubscriber(0x020000000000ull).ok());
    auto again = (*pool.value)->Allocate(0x02AA00000001ull); // a released address can be leased again
    CHECK(again.ok() && *again.value != leased[0x020000000000ull + 12]);
    t = mon.Tick(1075ull * 1000000000ull);
    CHECK(t.ok() && gauge[3] == 1000 / 16 && mon.Level(3) == dhcp::PoolLevel::Ok);
}

int main(int argc, char **argv) {
    const bool gpu = argc > 1 && !strcmp(argv[1], "gpu");
    if (gpu) {
        test_gpu_two_shards_leases();
        test_gpu_server_census_and_cleanup();
    } else {
        test_sizes();
        test_pool_monitor();
        test_cleanup_loop();
        test_merge();
    }
    if (failures) return 1;
    printf("ok\n");
    return 0;
}
