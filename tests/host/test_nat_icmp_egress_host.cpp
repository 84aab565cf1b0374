// Tests of the host side of upstream ICMP error translation (bng_nat_icmp_errors_egress_enable):
// nat::ManagerConfig::EnableUpstreamICMPErrorTranslation applied by nat::Manager::Start, and
// shard::Router::NatICMPErrorsEgressEnable reaching every shard (bng_host.hpp, bng_shard.hpp).
// `test_nat_icmp_egress_host cpu` needs no device: the NULL-context check.  `test_nat_icmp_egress_host gpu` observes
// the flag through its effect: a subscriber's UDP flow is SNATed by nat44_egress, the remote's reply is DNATed by
// nat44_ingress, and the subscriber's port unreachable quoting that reply leaves through nat44_egress from the public
// address, quoting the public address and port, when translation is on; keyed by its bytes 4-5 as before when off.
#include <cerrno>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

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
    b->wire_order_keys = true; // addresses as the programs read them off the wire
    return b;
}

static void put16(uint8_t *p, uint16_t v) { p[0] = (uint8_t)(v >> 8), p[1] = (uint8_t)v; }

// An Ethernet + IPv4 (ihl 5) header at f, protocol proto, from src to dst (network order bytes), total length tl.
static void ipv4(uint8_t *f, const uint8_t *src, const uint8_t *dst, uint8_t proto, uint16_t tl) {
    f[12] = 0x08, f[13] = 0x00, f[14] = 0x45, f[22] = 64, f[23] = proto;
    put16(f + 16, tl);
    memcpy(f + 26, src, 4);
    memcpy(f + 30, dst, 4);
}

// The subscriber's ICMP error (type, code 3) about the frame r it received (r: a frame as nat44_ingress left it):
// from r's destination to r's source, quoting r's IPv4 header and its first qlen - 20 bytes.  Frame length 42 + qlen.
static void sub_error(uint8_t *f, const uint8_t *r, uint8_t type, uint32_t qlen) {
    memcpy(f, r + 6, 6), memcpy(f + 6, r, 6);
    ipv4(f, r + 30, r + 26, 1, (uint16_t)(28 + qlen));
    f[34] = type, f[35] = 3;
    memcpy(f + 42, r + 14, qlen);
}

static int run(bng_ctx *c, const char *prog, std::vector<uint8_t> &frames, uint32_t n, uint32_t stride,
               std::vector<uint32_t> len, uint64_t now, std::vector<uint8_t> *verdict_out = nullptr) {
    std::vector<uint8_t> verdict(n);
    bng_batch bt{};
    bt.pkts = frames.data(), bt.len = len.data(), bt.verdict = verdict.data(), bt.n = n, bt.stride = stride;
    bt.mem = BNG_MEM_HOST, bt.arena_bytes = (uint32_t)(frames.size() / 16), bt.now_ns = now;
    const int rc = bng_prog_run(c, bng_prog_id(c, prog), &bt);
    if (verdict_out) *verdict_out = verdict;
    return rc;
}

// 100.64.0.<s>:40000 sends a UDP frame to 8.8.8.8:53 through nat44_egress, the reply comes back through
// nat44_ingress, and the subscriber's port unreachable quoting that reply goes through nat44_egress.  Returns whether
// it left translated: from the public address, quoting the public address and port.
static bool error_leaves_translated(bng_ctx *c, uint8_t s) {
    const uint8_t sub[4] = {100, 64, 0, s}, dns[4] = {8, 8, 8, 8};
    std::vector<uint8_t> up(64);
    ipv4(up.data(), sub, dns, 17, 50);
    put16(&up[34], 40000);
    put16(&up[36], 53);
    put16(&up[38], 30);
    CHECK(run(c, "nat44_egress", up, 1, 64, {64}, 1000000000ull) == 0);
    CHECK(memcmp(&up[26], sub, 4) != 0); // SNATed
    uint8_t pub[4], pport[2];
    memcpy(pub, &up[26], 4), memcpy(pport, &up[34], 2);
    std::vector<uint8_t> down(64);
    ipv4(down.data(), dns, pub, 17, 50);
    memcpy(&down[34], &up[36], 2), memcpy(&down[36], pport, 2);
    put16(&down[38], 30);
    CHECK(run(c, "nat44_ingress", down, 1, 64, {64}, 1500000000ull) == 0);
    CHECK(memcmp(&down[30], sub, 4) == 0); // DNATed
    std::vector<uint8_t> err(128);
    sub_error(err.data(), down.data(), 3, 28);
    CHECK(run(c, "nat44_egress", err, 1, 128, {70}, 2000000000ull) == 0);
    const bool outer = memcmp(&err[26], pub, 4) == 0, inner = memcmp(&err[58], pub, 4) == 0;
    const bool port = memcmp(&err[64], pport, 2) == 0, rest = err[38] == 0 && err[39] == 0; // bytes 4-5 untouched
    CHECK(outer);          // SNATed either way (off: by a session keyed on bytes 4-5)
    CHECK(inner == port);
    CHECK(inner || memcmp(&err[58], sub, 4) == 0); // off: the quote still names the subscriber
    return inner && port && rest;
}

static bool launched(bng_ctx *c, const char *name) {
    std::vector<char> buf(1 << 16);
    int64_t n = bng_prof_read(c, buf.data(), buf.size());
    return n > 0 && std::string(buf.data(), (size_t)n).find(name) != std::string::npos;
}

static void test_null() {
    CHECK(bng_nat_icmp_errors_egress_enable(nullptr, 1) == -EINVAL && bng_nat_icmp_errors_egress_enable(nullptr, 0) == -EINVAL);
}

static void test_gpu_manager() {
    for (bool on : {false, true}) {
        auto be = open_ctx(0, 1);
        if (!be->ctx) return;
        nat::ManagerConfig cfg;
        cfg.Interface = "eth0", cfg.Backend_ = be, cfg.PortsPerSubscriber = 64, cfg.EnableUpstreamICMPErrorTranslation = on;
        auto m = nat::Manager::NewManager(cfg);
        CHECK(m.ok());
        CHECK(!(*m)->Start());
        CHECK(!(*m)->AddPublicIP(IPv4(203, 0, 113, 1)));
        for (uint8_t s : {1, 2}) {
            CHECK((*m)->AllocateNAT(IPv4(100, 64, 0, s)).ok());
            CHECK(error_leaves_translated(be->ctx, s) == on);
        }
    }
}

static void test_gpu_router() {
    auto dir = std::make_shared<shard::Directory>(2, 1024, 64);
    std::vector<std::shared_ptr<Backend>> shards = {open_ctx(0, 2), open_ctx(1, 2)};
    if (!shards[0]->ctx || !shards[1]->ctx) return;
    shard::Router r(shards, dir);
    std::vector<uint8_t> f(64);
    auto probe = [&](const char *prog, const char *name) {
        bool all = true;
        for (auto &s : shards) {
            CHECK(bng_prof_enable(s->ctx, 1) == 0);
            CHECK(run(s->ctx, prog, f, 1, 64, {64}, 1000000000ull) == 0);
            all = all && launched(s->ctx, name);
            CHECK(bng_prof_enable(s->ctx, 0) == 0);
        }
        return all;
    };
    const char *progs[3][2] = {{"nat44_egress", "(k_resolve<true, false, false, icmperr>)"},
                               {"pipeline_up", "(k_resolve<true, true, false, icmperr>)"},
                               {"pipeline_tc", "(k_resolve<true, true, false, tc, icmperr>)"}};
    for (auto &p : progs) CHECK(!probe(p[0], "icmperr>")); // off by default
    CHECK(r.NatICMPErrorsEgressEnable(true) == 0);
    for (auto &p : progs) CHECK(probe(p[0], p[1]));
    CHECK(!probe("nat44_ingress", "icmperr>")); // the downstream switch is a separate one
    CHECK(r.NatICMPErrorsEgressEnable(false) == 0);
    for (auto &p : progs) CHECK(!probe(p[0], "icmperr>"));
}

// One context against two shards behind a Router with the flag on: every subscriber's flows go upstream to its
// shard (SteerUpstream), the replies come back through SteerDownstream, and the subscribers' ICMP errors quoting those
// replies, of several lengths, types and kinds, are steered one by one by SteerUpstream.  The shards' frames,
// verdicts and NAT counters add up to the one context's.
static void test_gpu_sharded() {
    const uint32_t world = 2, n_subs = 16;
    auto dir = std::make_shared<shard::Directory>(world, 1024, 64);
    std::vector<std::shared_ptr<Backend>> shards = {open_ctx(0, world), open_ctx(1, world)};
    auto whole = open_ctx(0, 1);
    if (!shards[0]->ctx || !shards[1]->ctx || !whole->ctx) return;
    shard::Router r(shards, dir);
    CHECK(r.NatICMPErrorsEgressEnable(true) == 0);
    CHECK(bng_nat_icmp_errors_egress_enable(whole->ctx, 1) == 0);
    std::vector<std::shared_ptr<Backend>> all = {shards[0], shards[1], whole};
    std::vector<std::shared_ptr<nat::Manager>> mgr;
    for (auto &b : all) {
        nat::ManagerConfig cfg;
        cfg.Interface = "eth0", cfg.Backend_ = b, cfg.PortsPerSubscriber = 64;
        auto m = *nat::Manager::NewManager(cfg).value;
        CHECK(!m->Start());
        CHECK(!m->AddPublicIP(IPv4(203, 0, 113, 1)));
        mgr.push_back(m);
    }
    static const uint8_t dns[4] = {8, 8, 8, 8};
    const uint32_t per = 4; // UDP with a checksum, UDP without, TCP, ICMP echo
    std::vector<uint8_t> up(n_subs * per * 64);
    std::vector<uint64_t> mac(n_subs);
    for (uint32_t s = 0; s < n_subs; s++) {
        const uint8_t ip[4] = {100, 64, 1, (uint8_t)(s + 1)};
        uint32_t key;
        memcpy(&key, ip, 4);
        mac[s] = 0x020000000100ull + s;
        dir->Learn(mac[s], key);
        for (auto &m : mgr) {
            auto a = m->AllocateNAT(IPv4(100, 64, 1, (uint8_t)(s + 1)));
            CHECK(a.ok());
            if (&m == &mgr.back() && a.ok()) {
                uint32_t pub;
                memcpy(&pub, To4(a.value->PublicIP), 4);
                dir->AddBlock(pub, a.value->PortStart, key);
            }
        }
        for (uint32_t k = 0; k < per; k++) {
            uint8_t *f = &up[(s * per + k) * 64];
            for (int j = 0; j < 6; j++) f[6 + j] = (uint8_t)(mac[s] >> (40 - 8 * j));
            const uint8_t proto = k < 2 ? 17 : (k == 2 ? 6 : 1);
            ipv4(f, ip, dns, proto, 50);
            put16(f + 34, (uint16_t)(40000 + k));
            if (proto == 1) {
                f[34] = 8, f[35] = 0;
                put16(f + 38, (uint16_t)(42000 + s));
            } else {
                put16(f + 36, proto == 6 ? 443 : 53);
                put16(f + (proto == 6 ? 50 : 40), k == 1 ? 0 : (uint16_t)(0x1234 + s)); // UDP k = 1: no checksum
            }
        }
    }
    const uint32_t n_up = n_subs * per;
    std::vector<uint8_t> snat = up;
    CHECK(run(whole->ctx, "nat44_egress", snat, n_up, 64, std::vector<uint32_t>(n_up, 64), 1000000000ull) == 0);
    for (uint32_t i = 0; i < n_up; i++) {
        std::vector<uint8_t> one(up.begin() + i * 64, up.begin() + (i + 1) * 64);
        const uint32_t k = dir->SteerUpstream(one.data(), 64);
        CHECK(run(shards[k]->ctx, "nat44_egress", one, 1, 64, {64}, 1000000000ull) == 0);
        CHECK(memcmp(one.data(), &snat[i * 64], 64) == 0);
    }
    // the replies, DNATed by the shard of their public port
    std::vector<uint8_t> rep(n_up * 64);
    for (uint32_t i = 0; i < n_up; i++) {
        const uint8_t *q = &snat[i * 64];
        uint8_t *f = &rep[i * 64];
        memcpy(f, q, 64);
        memcpy(f, q + 6, 6), memcpy(f + 6, q, 6);
        memcpy(f + 26, q + 30, 4), memcpy(f + 30, q + 26, 4);
        if (q[23] == 1)
            f[34] = 0;
        else
            memcpy(f + 34, q + 36, 2), memcpy(f + 36, q + 34, 2);
    }
    std::vector<uint8_t> dnat = rep;
    CHECK(run(whole->ctx, "nat44_ingress", dnat, n_up, 64, std::vector<uint32_t>(n_up, 64), 1500000000ull) == 0);
    for (uint32_t i = 0; i < n_up; i++) {
        std::vector<uint8_t> one(rep.begin() + i * 64, rep.begin() + (i + 1) * 64);
        const uint32_t k = dir->SteerDownstream(one.data(), 64, 0);
        CHECK(run(shards[k]->ctx, "nat44_ingress", one, 1, 64, {64}, 1500000000ull) == 0);
        CHECK(memcmp(one.data(), &dnat[i * 64], 64) == 0);
    }
    // the subscribers' errors about the replies they received
    std::vector<uint8_t> errs;
    std::vector<uint32_t> lens;
    for (uint32_t i = 0; i < n_up; i++) {
        for (uint32_t len = 34 + i % 3; len <= 92; len += 3) {
            uint8_t f[128] = {0};
            sub_error(f, &dnat[i * 64], (uint8_t)(len % 2 ? 11 : (len % 3 ? 3 : 12)), 50); // the whole quoted packet
            if (len % 7 == 0) f[61] ^= 1;      // the quote is not addressed to the error's source
            if (len % 11 == 0) f[65] ^= 0x40;  // a quoted port no flow has
            errs.insert(errs.end(), f, f + 128);
            lens.push_back(len);
        }
    }
    const uint32_t n = (uint32_t)lens.size();
    std::vector<uint8_t> one = errs, want_v;
    CHECK(run(whole->ctx, "nat44_egress", one, n, 128, lens, 2000000000ull, &want_v) == 0);
    uint32_t to[2] = {0, 0}, translated = 0;
    for (uint32_t i = 0; i < n; i++) {
        const std::vector<uint8_t> exact(errs.begin() + i * 128, errs.begin() + i * 128 + lens[i]); // len bytes
        const uint32_t k = dir->SteerUpstream(exact.data(), lens[i]);
        to[k]++;
        std::vector<uint8_t> f(errs.begin() + i * 128, errs.begin() + (i + 1) * 128), v;
        CHECK(run(shards[k]->ctx, "nat44_egress", f, 1, 128, {lens[i]}, 2000000000ull, &v) == 0);
        CHECK(memcmp(f.data(), &one[i * 128], 128) == 0);
        CHECK(v[0] == want_v[i]);
        translated += lens[i] >= 66 && memcmp(&one[i * 128 + 58], &one[i * 128 + 26], 4) == 0 &&
                      one[i * 128 + 26] == 203;
    }
    CHECK(to[0] > 0 && to[1] > 0);
    CHECK(translated > n_up);
    uint64_t st[3][13];
    for (int c = 0; c < 3; c++) {
        uint32_t key = 0;
        CHECK(bng_map_lookup(all[c]->ctx, bng_map_id(all[c]->ctx, "nat_stats_map"), &key, st[c]) == 0);
    }
    for (int j = 0; j < 13; j++) CHECK(st[0][j] + st[1][j] == st[2][j]);
}

int main(int argc, char **argv) {
    std::string mode = argc > 1 ? argv[1] : "cpu";
    test_null();
    if (mode == "gpu") {
        test_gpu_manager();
        test_gpu_router();
        test_gpu_sharded();
    }
    printf("%d checks, %d failed\n", g_checks, g_fail);
    return g_fail ? 1 : 0;
}
